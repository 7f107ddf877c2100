"""GPU: CUDA-graph replay on the configurations the TMA post-physics kernel does not take.  The warp-per-env kernel (env_step.cu) runs
20- and 50-step histories, shards that are not a multiple of 32 envs and `generic_kernel=True`; it reads the device step record of
dwbc_post_physics_step_device like the TMA kernel does, so a captured rollout (RolloutGraph) replays there too.

  * eager against replayed, bit for bit, on the workload of tools/history_bench.py at each such configuration (and the rough config on
    the TMA kernel): two PPO iterations and one DAgger iteration, rollout + compute_returns + update() / update_dagger(), the command
    curriculum and the mixing / priv-reg schedules moving, a push step inside the first rollout, resets, no library launch during a replay;
  * the two kernels in device-record mode against each other and against the eager host-argument call over 60 Philox steps;
  * one device-record call on the warp-per-env kernel against the host-argument call, on a push step and the step after it, at a
    50-step history and on a 33-env shard whose last CTA has one active warp.

Which kernel ran is read from derived_state column 27 (the TMA kernel's out-of-range history counter, always 0 after the warp-per-env
kernel), as in test_gpu_env_rollout.py.  A 20- or 50-step history (>= 1024 floats per row) takes the streaming form of the warp-per-env
kernel, a 10-step history its register form."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from dwbc_b200.config import WidowGo1Params
from test_gpu_cuda_graphs import ReplayLaunches, _tensors, assert_bitwise
from test_gpu_env import load_sim, make_core
from test_gpu_env_rollout import OOB_AGE

pytestmark = pytest.mark.gpu

T = 24                                   # rollout length: steps 131 .. 202 over three iterations; the push of step 150 is in the first
HP = dict(value_loss_coef=1.0, use_clipped_value_loss=True, clip_param=0.2, entropy_coef=0.0, num_learning_epochs=2, num_mini_batches=4,
          learning_rate=2e-4, gamma=0.99, lam=0.95, max_grad_norm=1.0, min_policy_std=[[0.15, 0.25, 0.25] * 4 + [0.2] * 3 + [0.05] * 3],
          mixing_schedule=[1.0, 1500, 4], priv_reg_coef_schedual=[0, 1, 1500, 4])
MOVING = {k + "_schedule": [0, 6] for k in ("lin_vel_x", "ang_vel_yaw", "tracking_ang_vel_yaw", "l", "p", "y")}   # moves at every update
CURRICULUM = (L.StepDevice.lin_vel_x.offset, C.sizeof(L.StepDevice))       # byte range of the curriculum block in the record


def workload(H, N, config, generic_kernel, precision):
    """tools/history_bench.py's workload at history_len H and N envs (bench.Workload's terrain layout for `rough`)."""
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.env import FusedWidowGo1Core
    from dwbc_b200.ppo import FusedPPO
    dev = "cuda:0"
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
    env = FusedWidowGo1Core(p, dev, state=st, seed=1000, sync_stats=False, generic_kernel=generic_kernel)
    env.common_step_counter = 130
    ac = FlatActorCritic(device=dev, seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=H, num_prop=76)
    alg = FusedPPO(ac, device=dev, precision=precision, **HP)
    alg.init_storage(N, T, [p.num_obs], [None], [p.num_actions])
    alg.counter = 1500
    alg.generator = torch.Generator(device=dev)
    alg.generator.manual_seed(7)
    g = torch.Generator(device=dev)
    g.manual_seed(31)
    base = {k: torch.from_numpy(v).to(dev) for k, v in synth.sim_state(p, 100, 1, rp_sigma=0.05, z_lo=0.327).items()}
    if p.terrain_curriculum:
        base["root_states"][:, 0, 0:2] += env.env_origins[:, 0:2]
    pool = []
    for _ in range(T):
        s = {k: (base[k] + torch.randn(base[k].shape, device=dev, generator=g) * 0.02 * base[k].abs().clamp(min=0.05)).contiguous()
             for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]
        s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        pool.append(s)
    env.set_obs_target(alg.storage.obs_row(0))
    return SimpleNamespace(p=p, env=env, alg=alg, pool=pool, obs=alg.storage.obs_row(0))


def eager_rollout(w, hist_encoding):
    """bench.Workload.rollout: the loop RolloutGraph captures."""
    env, alg, s = w.env, w.alg, w.alg.storage
    obs = w.obs
    if obs.data_ptr() != s.obs_row(0).data_ptr():
        s.obs_row(0).copy_(obs)
        obs = s.obs_row(0)
    for t in range(T):
        actions = alg.act(obs, obs, hist_encoding)
        env.bind_sim(**w.pool[t])
        env.set_obs_target(s.obs_row(t + 1))
        env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
        env.pre_physics_step(actions)
        env.post_physics_step()
        obs = env.obs_buf
        alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
    return obs


def run(H, N, config, generic_kernel, precision, graphs):
    from dwbc_b200.graphs import RolloutGraph
    w = workload(H, N, config, generic_kernel, precision)
    alg, env = w.alg, w.env
    alg.cuda_graphs = graphs
    rg = RolloutGraph(alg, env, physics=lambda t: env.bind_sim(**w.pool[t])) if graphs else None
    results, curriculum = [], []
    for dagger in (False, False, True):
        env.update_command_curriculum()
        curriculum.append(tuple(env.curriculum.lin_vel_x_ranges))
        obs = rg.run(w.obs, dagger) if graphs else eager_rollout(w, dagger)
        alg.compute_returns(obs)
        results.append(torch.tensor([alg.update_dagger()] if dagger else list(alg.update()), dtype=torch.float64))
        w.obs = obs
    assert len(set(curriculum)) == 3, curriculum        # the curriculum values of the step record moved at every iteration
    if graphs:
        assert len(rg._graphs) == 2                     # one rollout graph with and one without the history-encoder latent
    out = dict(losses=torch.cat(results), obs=w.obs.clone(), step_counter=torch.tensor(env.common_step_counter),
               adam_steps=torch.tensor([alg.optimizer.step, alg.hist_encoder_optimizer.step]))
    for prefix, obj in (("alg", alg), ("storage", alg.storage), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                        ("ac", alg.actor_critic), ("env", env)):
        out.update(_tensors(prefix, obj))
    out.update({f"episode.{k}": torch.as_tensor(v, dtype=torch.float64) for k, v in env.episode_stats(reset=False).items()})
    out.update({f"pool{t}.{k}": v.clone() for t, p in enumerate(w.pool) for k, v in p.items()})
    del w, rg
    torch.cuda.empty_cache()
    return out


# history_len, envs, config, generic_kernel, kernel that runs (True: TMA), precision
CASES = [(20, 1024, "flat", False, False, "tf32x3"),
         (50, 1000, "flat", False, False, "fp32"), (50, 1000, "flat", False, False, "tf32"), (50, 1000, "flat", False, False, "tf32x3"),
         (10, 1000, "flat", False, False, "tf32x3"),
         (10, 1024, "flat", True, False, "tf32x3"),
         (10, 1024, "rough", False, True, "tf32x3")]
IDS = ["h20-1024", "h50-1000-fp32", "h50-1000-tf32", "h50-1000-tf32x3", "h10-1000", "h10-1024-generic", "rough-h10-1024-tma"]


@pytest.mark.parametrize("H,N,config,generic_kernel,tma,precision", CASES, ids=IDS)
def test_graphs_replay_the_eager_bits(H, N, config, generic_kernel, tma, precision, monkeypatch):
    eager = run(H, N, config, generic_kernel, precision, False)
    counter = ReplayLaunches(monkeypatch)
    graphed = run(H, N, config, generic_kernel, precision, True)
    assert counter.replays == 6 and counter.moved == 0, (counter.replays, counter.moved)
    assert eager["losses"].isfinite().all()
    assert float(eager["env._stats"][0]) > 0                       # episodes ended (resets) during the three rollouts
    assert eager["losses"][3] != eager["losses"][10]                # the mixing schedule moved between the two PPO iterations
    age = eager["env._derived_state"][:, OOB_AGE]
    assert bool((age > 0).any()) if tma else not bool(age.any()), "the other post-physics kernel ran"
    assert_bitwise(eager, graphed)


# ---------------------------------------------------------------------------------------------- device records, kernel by kernel
def device_record(core):
    """A CUDA DwbcStepDevice holding core.step_record(), bound with set_device_step."""
    rec = core.step_record().cuda()
    core.set_device_step(rec)
    return rec


def record_step(rec):
    return int(rec[:8].cpu().numpy().view(np.uint64)[0])


def spoil_host_args(core):
    """Make the host's step, push decision and curriculum values wrong: a call with a device record must not read them."""
    core.common_step_counter += 7
    first, end = L.StepArgs.lin_vel_x.offset, L.StepArgs.generic_kernel.offset
    C.memset(C.addressof(core._args) + first, 0, end - first)


def outputs(core):
    return _tensors("env", core, skip=("_dev_step",))


def test_kernels_agree_on_device_records():
    """4096 envs, 10-step history: a TMA core and a generic_kernel=True core through dwbc_post_physics_step_device, each with its own
    record (step uploaded once, then only advanced on the device; curriculum block rewritten by a stream-ordered copy every 20 steps),
    against each other and against a TMA core on the host arguments, over 60 Philox steps from common_step_counter 140 (push at 150,
    time-outs).  Everything bit for bit; the generic kernel leaves the out-of-range history counter at 0."""
    from dwbc_b200.graphs import HostUpload
    seed, N, steps = 51, 4096, 60
    p = WidowGo1Params(num_envs=N, **MOVING)
    st = E.initial(p, seed)
    a, b, ref = make_core(p, st, seed=77), make_core(p, st, seed=77, generic_kernel=True), make_core(p, st, seed=77)
    for c in (a, b, ref):
        c.common_step_counter = 140
    recs = [device_record(a), device_record(b)]
    uploads = [HostUpload(), HostUpload()]
    n_reset = n_push = 0
    for t in range(1, steps + 1):
        if t % 20 == 1:
            for c in (a, b, ref):
                c.update_command_curriculum()
            for c, rec, up in zip((a, b), recs, uploads):
                up(rec[CURRICULUM[0]:], c.step_record()[CURRICULUM[0]:])
                spoil_host_args(c)
        sim = synth.sim_state(p, seed, t)
        for c in (a, b, ref):
            load_sim(c, p, sim)
            c.post_physics_step()
        n_push += int(ref._pushed)
        n_reset += int(ref.reset_buf.sum())
        oa, ob, oref = outputs(a), outputs(b), outputs(ref)
        assert_bitwise(oa, oref)
        da, db = oa.pop("env._derived_state"), ob.pop("env._derived_state")
        assert bool((da[:, OOB_AGE] > 0).any()) and not bool(db[:, OOB_AGE].any()), f"step {t}: a kernel other than the expected one ran"
        keep = [i for i in range(da.shape[1]) if i != OOB_AGE]
        assert torch.equal(da[:, keep], db[:, keep]), f"step {t}"
        assert_bitwise(oa, ob)
    assert n_push == 1 and n_reset > 0
    assert record_step(recs[0]) == record_step(recs[1]) == 141 + steps


@pytest.mark.parametrize("H,N,push_robots", [(50, 1000, True), (10, 33, True), (10, 33, False)], ids=["h50-1000", "h10-33", "h10-33-no-push"])
def test_device_record_equals_host_arguments_on_warp_per_env_kernel(H, N, push_robots):
    """Steps 150 (push) and 151 on the warp-per-env kernel: a call whose record holds what the host would pass gives the bits of the
    host-argument call, and advances record.step by exactly 1.  With push_robots off the record's push_interval is 0: nothing is pushed
    at step 150, so the base velocities of the envs that did not reset are still the simulator's."""
    seed = 61
    p = WidowGo1Params(num_envs=N, history_len=H, push_robots=push_robots)
    st = E.initial(p, seed)
    host, dev = make_core(p, st, seed=5), make_core(p, st, seed=5)
    host.common_step_counter = dev.common_step_counter = 149
    rec = device_record(dev)
    assert int(L.StepDevice.from_buffer_copy(bytes(rec.cpu().numpy())).push_interval) == (150 if push_robots else 0)
    spoil_host_args(dev)
    for t, push in ((1, push_robots), (2, False)):
        sim = synth.sim_state(p, seed, t)
        for c in (host, dev):
            load_sim(c, p, sim)
            c.post_physics_step()
        assert host._pushed == push
        assert record_step(rec) == 150 + t
        assert not bool(host._derived_state[:, OOB_AGE].any()), "the TMA kernel ran"
        assert_bitwise(outputs(host), outputs(dev))
        kept = ~dev.reset_buf.cpu()
        moved = ~torch.from_numpy(sim["root_states"][:, 0, 7:9] == dev.root_states[:, 7:9].cpu().numpy()).all(dim=1)
        assert bool(kept.any()) and bool(moved[kept].any()) == push, f"step {149 + t}: push {push}"
