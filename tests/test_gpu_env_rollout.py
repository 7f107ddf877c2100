"""The post-physics step over whole rollouts: both kernels against the CPU oracle with observations beyond clip_observations, at
shard sizes that take the generic kernel, and the two kernels against each other in production (Philox) mode.

The TMA kernel (env_step_v2.cu) re-emits the stored history as obs[:, 100:] with a bulk copy of the UNCLIPPED rows and patches the
row with a clipped copy only while a per-env counter (derived_state column 27: how many of the most recent history rows are known to
lie within +-clip_observations) is below history_len.  Synthetic states never leave +-100, so these tests push single observation
columns out of range on a schedule that walks the counter through 0 .. H and back, and check the counter itself against a model.
The generic kernel (env_step.cu) always clips and always leaves the counter at 0, which is how every test checks which kernel ran."""
import math

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import synth
from dwbc_b200.config import WidowGo1Params
from oracle import env_oracle as EO
from test_gpu_env import FTOL, load_sim, make_core

pytestmark = pytest.mark.gpu
H = 10                    # history_len of every config here
OOB_AGE = 27              # derived_state column DWBC_DS_OOB_AGE
CTA = 16                  # envs per CTA of the TMA kernel (V2_E)
JOINT = 3                 # a leg joint (IG order); the waist joint (num_dofs - 8) is wrapped to +-pi and cannot leave the range


def params(name, N, clip=None):
    kw = dict(E.ENV_CONFIGS[name] if name in E.ENV_CONFIGS else E.BRANCH_CASES[name])
    if clip is not None:
        kw["clip_observations"] = clip
    return WidowGo1Params(num_envs=N, **kw)


# ---------------------------------------------------------------------------------------------- injected out-of-range events
class Schedule:
    """Edits of the per-step sim dict, applied identically for the kernel and the oracle.
    events[t] = [(env, kind, sign)]: one observation column of `env` beyond +-100 at step t --
      'ang' base angular velocity (obs scale 1.0): 150 rad/s about the base z axis;
      'vel' joint JOINT's velocity (obs scale 0.05): 2500 rad/s;
      'pos' joint JOINT's position: 150 rad from its default.
    resets[t] = [env]: the env is dropped below term_z so that it terminates at step t.
    Every env in `alive` is otherwise kept from terminating: upright (roll = pitch = 0) at z = 0.45, no force on the termination
    contact bodies (time-outs are avoided by picking envs with short initial episodes)."""

    def __init__(self):
        self.events, self.resets, self.alive = {}, {}, set()

    def event(self, t, env, kind, sign):
        self.events.setdefault(t, []).append((env, kind, sign))
        self.alive.add(env)

    def reset(self, t, env):
        self.resets.setdefault(t, []).append(env)
        self.alive.add(env)

    def apply(self, p, sim, t):
        N, nd = p.num_envs, p.num_dofs
        root, cf = sim["root_states"], sim["contact_forces"]
        dof = sim["dof_state"].reshape(N, nd, 2)
        for e in self.alive:
            yaw = 0.3 + 0.05 * (e % 7)
            root[e, 0, 2] = 0.45
            root[e, 0, 3:7] = (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))
            cf[e, p.termination_contact_indices, :] = 0.0
        for e in self.resets.get(t, ()):
            root[e, 0, 2] = 0.2
        for e, kind, sign in self.events.get(t, ()):
            if kind == "ang":
                root[e, 0, 10:13] = (0.0, 0.0, 150.0 * sign)
            elif kind == "vel":
                dof[e, JOINT, 1] = 2500.0 * sign
            else:
                dof[e, JOINT, 0] = p.default_dof_pos[JOINT] + 150.0 * sign


def add_schedule(s, ep0, groups, t0=0):
    """Events in three 16-env CTAs `groups` (several event envs per CTA), steps t0+1 .. t0+35:
    (a) one event, then >= H + 1 quiet steps; (b) two events H - 1 steps apart (and an event right after the counter returned to H);
    (c) an event on the first step of an episode and one on the reset step itself; all three column kinds, both signs."""
    def pick(g, k):
        c = [e for e in range(CTA * g, CTA * g + CTA) if 10 <= ep0[e] <= 400]     # no time-out within 60 steps
        assert len(c) >= k, f"CTA {g}: only {len(c)} envs with a short initial episode"
        return c[:k]
    a1, a2, b1, c1, c2 = pick(groups[0], 5)
    s.event(t0 + 2, a1, "ang", +1)
    s.event(t0 + 3, a2, "vel", -1)
    s.event(t0 + 4, b1, "pos", +1)
    s.event(t0 + 4 + H - 1, b1, "pos", +1)
    s.reset(t0 + 6, c1)
    s.event(t0 + 7, c1, "vel", +1)                 # first step of the new episode: the history is filled with the out-of-range row
    s.reset(t0 + 8, c2)
    s.event(t0 + 8, c2, "ang", -1)                 # reset step: the observation keeps the pre-reset angular velocity (WG:879)
    a3, b2, b3 = pick(groups[1], 3)
    s.event(t0 + 5, a3, "pos", -1)
    s.event(t0 + 2, b2, "ang", +1)
    s.event(t0 + 2 + H - 1, b2, "ang", +1)
    s.event(t0 + 2 + 2 * H, b2, "vel", -1)         # the counter is back at H: fast path, then out of range again
    s.event(t0 + 10, b3, "vel", -1)
    s.event(t0 + 10 + H - 1, b3, "vel", +1)
    s.event(t0 + 10 + H, b3, "pos", -1)            # consecutive events
    a4, c3, a5 = pick(groups[2], 3)
    s.event(t0 + 1, a4, "pos", +1)
    s.reset(t0 + 15, c3)
    s.event(t0 + 16, c3, "pos", -1)
    s.event(t0 + 24, a5, "vel", +1)
    return s


# ---------------------------------------------------------------------------------------------- kernel identification
def next_age(age, prop, ep_len, clip):
    """Model of the TMA kernel's counter after a step: 0 if this step's proprioception row is out of range, H after a history fill
    (first step of an episode, reset), else one more (saturating at 1e6)."""
    oob = ~(prop.abs() <= clip).all(dim=1)
    return torch.where(oob, 0.0, torch.where(ep_len <= 1, float(H), torch.clamp(age + 1.0, max=1.0e6)))


def check_kernel(core, specialised, age, t):
    got = core._derived_state[:, OOB_AGE].cpu()
    if specialised:
        assert bool((age > 0).any()), "no in-range env: the counter cannot tell the kernels apart"
        assert torch.equal(got, age), f"step {t}: the TMA kernel's out-of-range counter differs from the model (or another kernel ran)"
    else:
        assert not bool(got.any()), f"step {t}: nonzero out-of-range counter: the TMA kernel ran instead of the generic one"


# ---------------------------------------------------------------------------------------------- against the oracle
TASK_STATE = ("commands", "goal_timer", "ee_start_sphere", "ee_goal_sphere", "ee_goal_cart", "curr_ee_goal_sphere", "curr_ee_goal_cart",
              "ee_goal_orn_euler", "base_lin_vel", "base_ang_vel", "base_yaw_quat", "last_root_vel", "last_actions", "last_dof_vel",
              "feet_air_time", "ee_goal_delta_orn_euler")


def compare_with_oracle(core, orc, p, t, obs, rew, arew, rst):
    msg = f"step {t}"
    np.testing.assert_array_equal(core.reset_buf.cpu().numpy(), rst.numpy(), err_msg=f"reset {msg}")
    np.testing.assert_array_equal(core.time_out_buf.cpu().numpy(), orc.s.time_out_buf.numpy(), err_msg=f"time_out {msg}")
    np.testing.assert_array_equal(core.episode_length_buf.cpu().numpy(), orc.s.episode_length_buf.numpy(), err_msg=f"episode_length {msg}")
    np.testing.assert_allclose(core.obs_buf.cpu().numpy(), obs.numpy(), **FTOL, err_msg=f"obs {msg}")
    np.testing.assert_allclose(core.rew_buf.cpu().numpy(), rew.numpy(), **FTOL, err_msg=f"rew {msg}")
    np.testing.assert_allclose(core.arm_rew_buf.cpu().numpy(), arew.numpy(), **FTOL, err_msg=f"arm_rew {msg}")
    for k in TASK_STATE:
        np.testing.assert_allclose(getattr(core, k).cpu().numpy(), getattr(orc.s, k).numpy(), **FTOL, err_msg=f"{k} {msg}")
    np.testing.assert_allclose(core.obs_history_buf.cpu().numpy(), orc.s.obs_history_buf.numpy(), **FTOL, err_msg=f"history {msg}")
    np.testing.assert_allclose(core._root_states.cpu().numpy(), orc.s.root_states_full.numpy(), **FTOL, err_msg=f"root {msg}")
    np.testing.assert_allclose(core.dof_state.cpu().numpy(), orc.s.dof_state.numpy(), **FTOL, err_msg=f"dof {msg}")
    np.testing.assert_array_equal(core.action_history_buf.cpu().numpy(), orc.s.action_history_buf.numpy(), err_msg=f"action FIFO {msg}")
    np.testing.assert_array_equal(core.actions.cpu().numpy(), orc.s.actions.numpy(), err_msg=f"delayed actions {msg}")
    # episode sums, metric sums and, on reset steps, extras['episode'] (WG:743-750) with the tolerance of the golden test
    for k, v in orc.s.episode_sums.items():
        np.testing.assert_allclose(core.episode_sums[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=1e-6, err_msg=f"episode_sums[{k}] {msg}")
    for k, v in orc.s.episode_metric_sums.items():
        np.testing.assert_allclose(core.episode_metric_sums[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=1e-5, err_msg=f"metric {k} {msg}")
    if bool(rst.any()):
        ep = orc.extras["episode"]
        np.testing.assert_allclose([float(core.extras["episode"][k]) for k in ep], [float(ep[k]) for k in ep], rtol=1e-4, atol=1e-6,
                                   err_msg=f"extras['episode'] {msg}")
    if p.measure_heights:
        np.testing.assert_allclose(core.measured_heights.cpu().numpy(), orc.measured_heights.numpy(), rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(core.heights_obs.cpu().numpy(),
                                   EO.heights_obs(orc.root[:, 2], orc.measured_heights, p.obs_scale_height).numpy(), rtol=1e-6, atol=1e-6)
    if p.terrain_curriculum:
        np.testing.assert_array_equal(core.terrain_levels.cpu().numpy(), orc.s.terrain_levels.numpy(), err_msg=f"terrain level {msg}")
        np.testing.assert_array_equal(core.env_origins.cpu().numpy(), orc.s.env_origins.numpy(), err_msg=f"env origins {msg}")


def rollout_vs_oracle(p, seed, steps, specialised, generic_kernel=False, schedule=None, counter0=140):
    """Kernel and oracle over `steps` table-mode steps; returns the oracle's per-step record (out-of-range rows, episode lengths,
    resets) as [steps, N] tensors."""
    st = E.initial(p, seed)
    core = make_core(p, st, generic_kernel=generic_kernel)
    orc = EO.EnvOracle(p, E.oracle_state(p, st))
    rt = E.runtime(p)
    core.common_step_counter = orc.common_step_counter = counter0
    age = torch.zeros(p.num_envs)
    rec = dict(oob=[], ep_len=[], reset=[])
    for t in range(1, steps + 1):
        sim = E.sim_state(p, seed, t, orc.s.env_origins)
        if schedule is not None:
            schedule.apply(p, sim, t)
        load_sim(core, p, sim)
        E.load_sim_into_oracle(orc, p, sim)
        tab = torch.from_numpy(synth.rand_table(p, seed, t))
        obs, rew, arew, rst, _ = orc.post_physics_step(tab, rt)
        core.post_physics_step(tab.cuda())
        compare_with_oracle(core, orc, p, t, obs, rew, arew, rst)
        age = next_age(age, orc.s.prop, orc.s.episode_length_buf, p.clip_observations)
        check_kernel(core, specialised, age, t)
        rec["oob"].append(~(orc.s.prop.abs() <= p.clip_observations).all(dim=1))
        rec["ep_len"].append(orc.s.episode_length_buf.clone())
        rec["reset"].append(rst.clone())
    return {k: torch.stack(v) for k, v in rec.items()}


def coverage(rec):
    """Number of envs that went through each case of the counter (from the oracle's record):
    a: out of range, then H + 1 steps in range without a reset; b: out of range twice, H - 1 steps apart, no reset between;
    c: out of range on a step that fills the history (first step of an episode or a reset); d: CTAs with >= 2 such envs."""
    oob, ep_len, rst = rec["oob"], rec["ep_len"], rec["reset"]
    T, N = oob.shape
    a, b = torch.zeros(N, dtype=torch.bool), torch.zeros(N, dtype=torch.bool)
    for s in range(T):
        if s + H + 1 < T:
            a |= oob[s] & ~(oob[s + 1:s + H + 2] | rst[s + 1:s + H + 2]).any(0)
        if s + H - 1 < T:
            b |= oob[s] & oob[s + H - 1] & ~rst[s + 1:s + H].any(0)
    c = (oob & (ep_len <= 1)).any(0)
    per_cta = torch.bincount(torch.nonzero(oob.any(0)).flatten() // CTA, minlength=(N + CTA - 1) // CTA)
    return dict(a=int(a.sum()), b=int(b.sum()), c=int(c.sum()), d=int((per_cta >= 2).sum()), ctas=int((per_cta >= 1).sum()))


ROLLOUT_CASES = [(1024, False, True), (1024, True, False), (1000, False, False)]       # N, generic_kernel, specialised (expected)


@pytest.mark.parametrize("N,generic_kernel,specialised", ROLLOUT_CASES, ids=["1024-tma", "1024-generic", "1000-generic"])
@pytest.mark.parametrize("name", ["flat", "full"])
def test_rollout_with_out_of_range_observations_matches_oracle(name, N, generic_kernel, specialised):
    """36 steps with single observation columns pushed beyond +-100: obs (clipped), history (unclipped) and every output against
    the oracle at every step; the schedule must really have produced each case of the TMA kernel's counter."""
    seed = 21
    p = params(name, N)
    sched = add_schedule(Schedule(), synth.initial_env_state(p, seed)["episode_length_buf"], groups=(5, 23, 47))
    rec = rollout_vs_oracle(p, seed, 36, specialised, generic_kernel, sched)
    cov = coverage(rec)
    print(f"coverage {name} N={N} {'tma' if specialised else 'generic'}: {cov}")
    assert cov["a"] >= 5 and cov["b"] >= 3 and cov["c"] >= 3 and cov["d"] >= 3 and cov["ctas"] >= 3, cov
    assert int(rec["oob"].sum()) == sum(len(v) for v in sched.events.values())   # only the injected rows are out of range


@pytest.mark.parametrize("N,specialised", [(512, True), (500, False)], ids=["512-tma", "500-generic"])
@pytest.mark.parametrize("name", ["flat", "full"])
def test_rollout_with_dense_clipping_matches_oracle(name, N, specialised):
    """clip_observations = 1: most envs leave the range on most steps, in every column kind, across resets; 30 steps."""
    p = params(name, N, clip=1.0)
    rec = rollout_vs_oracle(p, 31, 30, specialised)
    oob = rec["oob"]
    assert 0.5 < float(oob.float().mean()) < 0.99                        # both paths taken, on most envs
    assert int((oob & (rec["ep_len"] <= 1)).sum()) > 0 and int((oob[1:] & ~oob[:-1]).sum()) > 0


@pytest.mark.parametrize("N,specialised", [(1, False), (3, False), (16, False), (33, False), (32, True)])
def test_shard_sizes_match_oracle(N, specialised):
    """Shards that are not a multiple of 32 take the generic kernel (16 is one TMA CTA's worth but still generic); 32 is exactly two
    TMA CTAs.  15 steps on `flat`, with out-of-range events on the last env."""
    p = params("flat", N)
    sched = Schedule()
    sched.event(2, N - 1, "ang", -1)
    sched.event(5, N - 1, "vel", +1)
    sched.event(9, N - 1, "pos", -1)
    rec = rollout_vs_oracle(p, 41, 15, specialised, schedule=sched)
    assert int(rec["oob"].sum()) == 3


# ---------------------------------------------------------------------------------------------- the two kernels, production mode
PHILOX_CASES = [("flat", False), ("full", False), ("flat", True)] + \
    [(name, False) for name in ("cart", "positive", "raw", "goals-0", "goals-3", "goals-11", "goals-16")]


@pytest.mark.parametrize("name,storage_rows", PHILOX_CASES, ids=[n + ("-storage-rows" if s else "") for n, s in PHILOX_CASES])
def test_tma_and_generic_kernel_agree_over_philox_rollout(name, storage_rows):
    """4096 envs, in-kernel Philox draws, 60 steps from common_step_counter 140 (push and command resampling at 150, time-outs),
    injected out-of-range events: every output and state buffer bit for bit (both kernels run the per-env code of
    env_step_common.cuh), episode sums and extras['episode'] included; only the TMA kernel's out-of-range counter column differs.
    Also on the config branches the TMA kernel takes (envstate.BRANCH_CASES: cart goals, positive-reward clip, unreordered DOFs with
    more contact bodies, goal searches with 0 .. 16 collision samples)."""
    seed, N, T = 51, 4096, 60
    p = params(name, N)
    st = E.initial(p, seed)
    a, b = make_core(p, st, seed=77), make_core(p, st, seed=77, generic_kernel=True)
    a.common_step_counter = b.common_step_counter = 140
    sched = Schedule()
    add_schedule(sched, st["episode_length_buf"], groups=(5, 23, 47))
    add_schedule(sched, st["episode_length_buf"], groups=(120, 201, 255), t0=22)
    stores = [torch.zeros(3, N, p.num_obs, device="cuda") for _ in range(2)] if storage_rows else None
    age = torch.zeros(N)
    n_timeout = n_reset = 0
    for t in range(1, T + 1):
        sim = E.sim_state(p, seed, t, a.env_origins)
        sched.apply(p, sim, t)
        for core, store in zip((a, b), stores or (None, None)):
            load_sim(core, p, sim)
            if store is not None:
                core.set_obs_target(store[t % 3])
            core.post_physics_step()
        msg = f"step {t}"
        for k in ("reset_buf", "time_out_buf", "episode_length_buf", "goal_timer", "last_contacts"):
            assert torch.equal(getattr(a, k), getattr(b, k)), f"{k} {msg}"
        if p.terrain_curriculum:
            assert torch.equal(a.terrain_levels, b.terrain_levels) and torch.equal(a.env_origins, b.env_origins), msg
        ds = [c._derived_state[:, [i for i in range(c._derived_state.shape[1]) if i != OOB_AGE]] for c in (a, b)]
        for k, x, y in (("obs", a.obs_buf, b.obs_buf), ("rew", a.rew_buf, b.rew_buf), ("arm_rew", a.arm_rew_buf, b.arm_rew_buf),
                        ("goal_state", a._goal_state, b._goal_state), ("derived_state", ds[0], ds[1]),
                        ("root", a._root_states, b._root_states), ("dof", a.dof_state, b.dof_state), ("history", a._hist, b._hist),
                        ("action_history", a.action_history_buf, b.action_history_buf), ("episode_sums", a._sums, b._sums)):
            assert torch.equal(x, y), f"{k} {msg}"
        if p.measure_heights:
            assert torch.equal(a.measured_heights, b.measured_heights), msg
            assert torch.equal(a.heights_obs, b.heights_obs), msg
        ea, eb = a.extras["episode"], b.extras["episode"]
        assert ea.keys() == eb.keys()
        np.testing.assert_array_equal([float(ea[k]) for k in ea], [float(eb[k]) for k in ea], err_msg=f"extras['episode'] {msg}")
        if storage_rows:
            assert a.obs_buf.data_ptr() == stores[0][t % 3].data_ptr()
        age = next_age(age, b.obs_history_buf[:, -1].cpu(), b.episode_length_buf.cpu(), p.clip_observations)
        check_kernel(a, True, age, t)
        check_kernel(b, False, age, t)
        n_timeout += int(a.time_out_buf.sum())
        n_reset += int(a.reset_buf.sum())
    assert n_timeout > 0 and n_reset > n_timeout


# ---------------------------------------------------------------------------------------------- obs target validation
def test_set_obs_target_rejects_unusable_tensors():
    """The kernels write 16-byte vectors into the observation target: a tensor they cannot use raises DwbcError before its pointer
    reaches the library (nothing is launched here), and leaves the previous target bound."""
    from dwbc_b200._lib import DwbcError
    from dwbc_b200.env import FusedWidowGo1Core
    N = 64
    p = params("flat", N)
    core = FusedWidowGo1Core(p, "cuda:0", state=E.initial(p, 1))
    n0 = int(core._lib.dwbc_launch_count())
    good = torch.zeros(2, N, p.num_obs, device="cuda")
    bad = {
        "float64": torch.zeros(N, p.num_obs, dtype=torch.float64, device="cuda"),
        "host": torch.zeros(N, p.num_obs),
        "transposed": torch.zeros(p.num_obs, N, device="cuda").t(),
        "offset by one float": torch.zeros(N * p.num_obs + 1, device="cuda")[1:].view(N, p.num_obs),
        "row stride not a multiple of 4": torch.zeros(N, p.num_obs + 1, device="cuda")[:, :p.num_obs],
        "too narrow": good[0, :, :p.num_obs - 4],
        "too few rows": good[0, :N - 1],
        "3-d": good,
    }
    core.set_obs_target(good[1])
    for what, t in bad.items():
        with pytest.raises(DwbcError):
            core.set_obs_target(t)
        assert core.obs_buf.data_ptr() == good[1].data_ptr(), what
        assert core._buf.obs_buf == good[1].data_ptr() and core._buf.obs_stride == p.num_obs, what
    core.set_obs_target(torch.zeros(N, p.num_obs + 4, device="cuda"))         # wider rows (e.g. storage with padding) are fine
    core.set_obs_target(None)
    assert core.obs_buf is core._obs_own and core._buf.obs_buf == core._obs_own.data_ptr()
    assert int(core._lib.dwbc_launch_count()) == n0
