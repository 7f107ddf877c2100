"""GPU: whole training iterations of the production loop against a teacher-forced float64 oracle, stage by stage.

The GPU side runs what the runner runs, unmodified: env.update_command_curriculum(), the rollout of bench.Workload.rollout (in-kernel Philox
draws, observations written into storage row t + 1 and rewards / dones into row t by the post-physics kernel, which adds the time-out
bootstrap itself), alg.compute_returns(obs_T) and alg.update() / update_dagger() without `indices`, so that the permutation comes from the
generator the action noise comes from.  Four iterations: PPO, PPO, DAgger (history-encoder rollout + update_dagger), PPO, with a FusedPPO
that tracks episodes and owns an explicit generator.  The schedules, both Adam states, the minimum std, obs row 0 of the next rollout and
the episode tracker carry from one iteration to the next.

The oracle side recomputes every stage from the GPU's outputs of the stage before it, cast to float64 (the env oracle runs in float32, as
in the env tests), so each comparison holds the tolerance its unit test states and errors do not compound; a glue error still shows,
because the oracle recomputes each row from the row it should have come from:
  * rng     -- a clone of the generator replays, in production order, one normal_((T, N, 18)) per rollout and one randperm(N * T) per update:
               the oracle's action noise and permutations;
  * act     -- PO.policy_act on obs row t and noise t against storage rows t of actions, values, log-probs, mu and sigma;
  * env     -- EnvOracle fed the GPU's action row t (clip, raisim2ig, delay FIFO), the sim state of step t and the uniform table of the step
               the kernel drew (dwbc_fill_uniform, tied to Philox itself by test_gpu_philox.py): obs row t + 1, rewards row t with the
               bootstrap PPO:133-134 on the GPU's values row t, dones row t;
  * gae     -- the critic on obs row T against the bootstrap values, then RS:136-150 on the GPU's rewards / values / dones;
  * update  -- PO.ppo_update / dagger_update from the GPU's parameters and Adam moments before the update, with the oracle's OWN Adam step
               counts and `counter`: the returned values and every parameter after the update (minimum std included);
  * episodes -- OnPolicyRunner's bookkeeping (OPR:140-154) on the oracle's rewards and dones against episode_buffers().
Every branch the join has is made to fire, and the test asserts that it did: time-outs inside rollouts, terminations, a push step, command
resampling, a curriculum that moves at every iteration, schedule values inside their ramps, and clipped ratios in the updates."""
import time

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200.config import WidowGo1Params
from oracle import env_oracle as EO
from oracle import ppo_oracle as PO
from test_episode_tracking_cpu import Restatement
from test_gpu_chain_shapes import TOL
from test_gpu_cuda_graphs_configs import MOVING
from test_gpu_env import FTOL
from test_gpu_env_rollout import Schedule

pytestmark = pytest.mark.gpu

T, SEED, ENV_SEED, STEP0, COUNTER0, TRACK = 8, 23, 1000, 146, 1500, 512
ITERATIONS = ("ppo", "ppo", "dagger", "ppo")
SIM_KEYS = ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")
INIT_STD = [[0.8, 1.0, 1.0] * 4 + [1.0] * 6]
# test_gpu_cuda_graphs_configs.HP with a minimum std above the initial hip std (0.85 > 0.8), so that enforce_min_std moves parameters
# after every update; the mixing and priv-reg ramps start at COUNTER0, so the four iterations see 0, 1/4, 2/4 (DAgger), 3/4 of them
HP = dict(value_loss_coef=1.0, use_clipped_value_loss=True, clip_param=0.2, entropy_coef=0.0, num_learning_epochs=2, num_mini_batches=4,
          learning_rate=2e-4, gamma=0.99, lam=0.95, max_grad_norm=1.0, min_policy_std=[[0.85, 0.25, 0.25] * 4 + [0.2] * 3 + [0.05] * 3],
          mixing_schedule=[1.0, COUNTER0, 4], priv_reg_coef_schedual=[0, 1, COUNTER0, 4])
# test_gpu_ppo.py / test_gpu_history_len.py: parameters after an update within 2e-5, fewer than 1e-4 of them beyond, none beyond 2 x lr
# (Adam moves an entry whose gradient is ~1e-8 by up to lr whatever the arithmetic); losses 2e-5 (relative above 1)
PARAM_ABS, PARAM_FRAC, LOSS_ABS = 2e-5, 1e-4, 2e-5
# test_gpu_ppo.py::test_gae_matches_oracle_full_size
RET_TOL, ADV_TOL = dict(rtol=1e-6, atol=1e-6), dict(rtol=1e-5, atol=2e-6)


# ---------------------------------------------------------------------------------------------- GPU side
class Production:
    """The runner's objects and loop.  The simulator of step t is a fixed set of device tensors (pool[t]) that physics(t) binds, refilled
    before each rollout, as bench.Workload does; a captured rollout binds the same tensors."""

    def __init__(self, config, N, precision, graphs, st):
        from dwbc_b200.actor_critic import FlatActorCritic
        from dwbc_b200.env import FusedWidowGo1Core
        from dwbc_b200.graphs import RolloutGraph
        from dwbc_b200.ppo import FusedPPO
        dev = "cuda:0"
        self.p = p = params(config, N)
        self.env = FusedWidowGo1Core(p, dev, state=st, seed=ENV_SEED, sync_stats=False)
        self.env.common_step_counter = STEP0
        ac = FlatActorCritic(device=dev, seed=0, init_std=INIT_STD, num_priv=24, num_hist=10, num_prop=76)
        self.alg = alg = FusedPPO(ac, device=dev, precision=precision, cuda_graphs=graphs, track_episodes=TRACK, **HP)
        alg.init_storage(N, T, [p.num_obs], [None], [p.num_actions])
        alg.counter = COUNTER0
        alg.generator = torch.Generator(device=dev)
        alg.generator.manual_seed(SEED)
        self.pool = [{k: torch.zeros(getattr(self.env, a).shape, device=dev) for k, a in
                      zip(SIM_KEYS, ("_root_states", "dof_state", "_rigid_body_state", "_contact_forces", "force_sensor_tensor", "torques"))}
                     for _ in range(T)]
        self.physics = lambda t: self.env.bind_sim(**self.pool[t])
        self.rg = RolloutGraph(alg, self.env, physics=self.physics) if graphs else None
        self.env.set_obs_target(alg.storage.obs_row(0))
        self.obs = alg.storage.obs_row(0)

    def rollout(self, hist_encoding):
        """bench.Workload.rollout (test_gpu_cuda_graphs_configs.eager_rollout), or its captured replay."""
        env, alg, s = self.env, self.alg, self.alg.storage
        if self.rg is not None:
            return self.rg.run(self.obs, hist_encoding)
        obs = self.obs
        if obs.data_ptr() != s.obs_row(0).data_ptr():
            s.obs_row(0).copy_(obs)
            obs = s.obs_row(0)
        for t in range(T):
            actions = alg.act(obs, obs, hist_encoding)
            self.physics(t)
            env.set_obs_target(s.obs_row(t + 1))
            env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
            env.pre_physics_step(actions)
            env.post_physics_step()
            obs = env.obs_buf
            alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
        return obs


def params(config, N):
    return WidowGo1Params(num_envs=N, **dict(E.ENV_CONFIGS[config], **MOVING))


def cpu64(x):
    return x.detach().to("cpu", torch.float64)


def named(ac, flat):
    return {n: cpu64(v) for n, v in ac.unflat(flat).items()}


# ---------------------------------------------------------------------------------------------- oracle side
class Stages:
    """Worst error per stage (printed) and every bound a stage missed (asserted at the end, all together, first stage first)."""

    def __init__(self):
        self.worst, self.failed, self.it = {}, [], 0

    def err(self, stage, got, want, atol, rtol=0.0):
        got, want = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(want, dtype=torch.float64)
        d = (got - want).abs()
        self.worst[stage] = max(self.worst.get(stage, 0.0), float(d.max()) if d.numel() else 0.0)
        over = d > atol + rtol * want.abs()
        if bool(over.any()):
            self.failed.append(f"iteration {self.it}, {stage}: {int(over.sum())} of {d.numel()} beyond atol {atol:g} rtol {rtol:g} (max {float(d.max()):.3g})")

    def exact(self, stage, got, want):
        if not torch.equal(torch.as_tensor(got), torch.as_tensor(want)):
            self.failed.append(f"iteration {self.it}, {stage}: not equal")

    def params(self, stage, got, want, lr):
        d = torch.cat([(got[n] - want[n]).abs().reshape(-1) for n in want])
        self.worst[stage] = max(self.worst.get(stage, 0.0), float(d.max()))
        frac = float((d > PARAM_ABS).double().mean())
        if frac >= PARAM_FRAC or float(d.max()) >= 2 * lr:
            self.failed.append(f"iteration {self.it}, {stage}: {frac:.2g} of the parameters beyond {PARAM_ABS:g}, max {float(d.max()):.3g} (2 x lr = {2 * lr:g})")

    def check(self, cond, what):
        if not cond:
            self.failed.append(what)


class Oracle:
    """The reference's state the GPU's must follow: the env oracle, `counter` and both Adam optimizers' step counts, the generator replay
    and the runner's episode bookkeeping."""

    def __init__(self, prod, st, hp):
        p, alg = prod.p, prod.alg
        self.p, self.hp, self.N = p, hp, p.num_envs
        self.env = EO.EnvOracle(p, E.oracle_state(p, st))
        self.env.common_step_counter = STEP0
        self.counter = COUNTER0
        names = [n for n, _ in alg.actor_critic.manifest]
        self.adam = PO.Adam(names, hp["learning_rate"])                                   # PPO:75
        self.hist_adam = PO.Adam([n for n in names if n.startswith(PO.HIST_PREFIX)], hp["learning_rate"])   # PPO:79
        self.rng = torch.Generator(device="cuda")
        self.rng.set_state(alg.generator.get_state())
        self.episodes = Restatement(self.N, TRACK)
        self.curriculum_count = 0
        self.cov = dict(time_outs=0, terminations=0, scheduled=0, pushes=0, resampled=0, clipped=0, rows=0, lin_vel_x=[], mixing=[],
                        priv_reg=[], rmax=[0.0, 0.0])

    def draw_noise(self):
        return cpu64(torch.empty(T, self.N, 18, device="cuda").normal_(generator=self.rng))

    def draw_perm(self):
        return torch.randperm(self.N * T, device="cuda", generator=self.rng).cpu()

    def rollout(self, S, snap, eps, hist_encoding, tol, sched_resets):
        """Stages act and env of one rollout; snap: the GPU's storage rows, the sim states and uniform tables of its steps."""
        p, orc = self.p, self.env
        self.curriculum_count += 1
        rt = E.runtime(p, self.curriculum_count)
        self.cov["lin_vel_x"].append(tuple(rt.lin_vel_x))
        P = snap["params"]
        for t in range(T):
            a = PO.policy_act(P, snap["obs"][t], eps[t], hist_encoding)
            for k, ref in (("actions", "actions"), ("values", "values"), ("log_prob", "actions_log_prob"), ("mean", "mu"), ("sigma", "sigma")):
                S.err(f"act {k}", snap[ref][t], a[k], tol)
            sim = dict(snap["sim"][t], policy_actions=snap["actions"][t].float().numpy())
            E.load_sim_into_oracle(orc, p, sim)
            self.cov["resampled"] += int(((orc.s.episode_length_buf + 1) % p.resample_interval == 0).sum())
            obs, rew, arew, rst, _ = orc.post_physics_step(snap["tables"][t], rt)
            to = orc.s.time_out_buf
            S.err("env obs", snap["obs"][t + 1], obs, FTOL["atol"], FTOL["rtol"])
            S.err("env rewards", snap["rewards"][t], PO.bootstrap_rewards(rew.double(), arew.double(), snap["values"][t], to, self.hp["gamma"]),
                  FTOL["atol"], FTOL["rtol"])
            S.exact("env dones", snap["dones"][t, :, 0], rst.to(torch.uint8))
            self.episodes.step(rew, arew, rst)
            self.cov["rmax"] = [max(m, float(r.abs().max())) for m, r in zip(self.cov["rmax"], (rew, arew))]
            self.cov["time_outs"] += int(to.sum())
            self.cov["terminations"] += int((rst & ~to).sum())
            self.cov["pushes"] += int(orc.pushed)
            step = orc.common_step_counter
            self.cov["scheduled"] += sum(int(rst[e]) for e in sched_resets.get(step, ()))

    def gae(self, S, snap):
        """RS:136-150 with the bootstrap of PPO:148-150."""
        last = PO.critic_values(snap["params"], snap["obs"][T])
        S.err("gae bootstrap values", snap["last_values"], last, TOL[snap["precision"]]["fwd"])
        ret, adv = PO.compute_returns(snap["rewards"], snap["values"], snap["dones"], snap["last_values"], self.hp["gamma"], self.hp["lam"])
        S.err("gae returns", snap["returns"], ret, RET_TOL["atol"], RET_TOL["rtol"])
        S.err("gae advantages", snap["advantages"], adv, ADV_TOL["atol"], ADV_TOL["rtol"])

    @staticmethod
    def _load_moments(opt, m, v):
        """The GPU's moments before the update; the step counts stay the oracle's own."""
        for n in opt.names:
            st = opt.state.setdefault(n, dict(step=0))
            st["m"], st["v"] = m[n].clone(), v[n].clone()

    def ppo(self, S, snap, perm):
        hp, P = self.hp, {n: v.clone() for n, v in snap["params"].items()}
        self._load_moments(self.adam, snap["m"], snap["v"])
        storage = {k: snap[k] for k in ("actions", "values", "returns", "advantages", "actions_log_prob")}
        storage["observations"] = snap["obs"][:T]
        mbs, nmb = perm.numel() // hp["num_mini_batches"], hp["num_mini_batches"]
        flat = {k: v.flatten(0, 1) for k, v in storage.items()}

        def record(k, Pk, G, when):           # clipped ratios of mini-batch k, from the parameters its loss saw
            if when == "pre_step":
                idx = perm[(k % nmb) * mbs:(k % nmb + 1) * mbs]
                lp = PO.log_prob2(PO.actor_mean(Pk, flat["observations"][idx]), Pk["std"], flat["actions"][idx])
                ratio = torch.exp(lp - flat["actions_log_prob"][idx])
                self.cov["clipped"] += int(((ratio - 1.0).abs() > hp["clip_param"]).sum())
                self.cov["rows"] += ratio.numel()

        logs = PO.ppo_update(P, self.adam, storage, perm, hp, self.counter, record=record)
        mean = lambda k: float(torch.stack([torch.as_tensor(l[k]) for l in logs]).mean())  # noqa: E731
        want = (mean("value"), mean("surrogate"), 0.0, logs[0]["mixing_ratio"], 0.0, mean("priv_reg"), logs[0]["priv_reg_coef"])
        res = snap["result"]
        for i, what in ((0, "value loss"), (1, "surrogate loss"), (5, "priv-reg loss")):
            S.err(f"update {what}", res[i], want[i], LOSS_ABS * max(1.0, abs(want[i])))
        for i, what in ((2, "torque loss"), (3, "mixing ratio"), (4, "torque weight"), (6, "priv-reg coefficient")):
            S.check(res[i] == want[i], f"update {what}: {res[i]} returned, the reference's schedule gives {want[i]} at counter {self.counter}")
        self.cov["mixing"].append(want[3])
        self.cov["priv_reg"].append(want[6])
        S.params("update parameters", snap["params_after"], P, hp["learning_rate"])
        self.counter += 1                                                                 # PPO:257-261
        return P

    def dagger(self, S, snap, perm):
        hp, P = self.hp, {n: v.clone() for n, v in snap["params"].items()}
        self._load_moments(self.hist_adam, snap["hist_m"], snap["hist_v"])
        losses = PO.dagger_update(P, self.hist_adam, dict(observations=snap["obs"][:T]), perm, hp)
        S.err("dagger loss", snap["result"][0], float(torch.stack(losses).mean()), LOSS_ABS)
        S.params("dagger parameters", snap["params_after"], P, hp["learning_rate"])
        # The reference's update_dagger (PPO:265-291) ends as update() does at PPO:257-261: storage.clear(), then counter += 1.  No golden
        # vector records the counter after it (tests/golden/make_golden.py:254-272 compares losses and parameters only); the next update's
        # mixing ratio and priv-reg coefficient, compared in ppo(), show whether the GPU advanced it.
        self.counter += 1


# ---------------------------------------------------------------------------------------------- the test
def initial_state(p):
    """E.initial, with the last 128 envs 0 .. 4T - 1 steps short of max_episode_length: time-outs at every step of the four rollouts."""
    st = E.initial(p, SEED)
    ep = st["episode_length_buf"]
    n = min(128, p.num_envs // 4)
    ep[-n:] = int(p.max_episode_length) - np.arange(n) % (len(ITERATIONS) * T)
    return st


def schedule(p, ep0):
    """Terminations on a schedule (test_gpu_env_rollout.Schedule): one env of a short initial episode dropped below term_z at each global
    step of the rollouts."""
    s = Schedule()
    cands = [e for e in range(p.num_envs - 128) if 10 <= ep0[e] <= 300]
    for i in range(len(ITERATIONS) * T):
        s.reset(STEP0 + 1 + i, cands[3 * i])
    return s


def snapshot(prod, sims, tables, precision):
    alg, s = prod.alg, prod.alg.storage
    snap = {k: cpu64(getattr(s, k)) for k in ("actions", "values", "actions_log_prob", "mu", "sigma", "rewards", "returns", "advantages")}
    snap.update(obs=cpu64(s._obs_all), dones=s.dones.cpu(), last_values=cpu64(alg._last_values), sim=sims, tables=tables, precision=precision)
    return snap


CASES = [("flat", 4096, "fp32", False), ("flat", 4096, "tf32x3", False), ("full", 1000, "fp32", False), ("full", 1000, "tf32x3", False),
         ("flat", 4096, "tf32x3", True)]


@pytest.mark.parametrize("config,N,precision,graphs", CASES, ids=["flat-4096-fp32", "flat-4096-tf32x3", "full-1000-fp32", "full-1000-tf32x3",
                                                                 "flat-4096-tf32x3-graphs"])
def test_training_iterations_match_the_oracle_stage_by_stage(config, N, precision, graphs):
    t_start = time.perf_counter()
    p = params(config, N)
    st = initial_state(p)
    sched = schedule(p, st["episode_length_buf"])
    prod = Production(config, N, precision, graphs, st)
    orc = Oracle(prod, st, HP)
    alg, env, ac, s = prod.alg, prod.env, prod.alg.actor_critic, prod.alg.storage
    S = Stages()
    prev_last_obs, step = None, STEP0
    for it, kind in enumerate(ITERATIONS):
        dagger, S.it = kind == "dagger", it
        # the oracle's draws, in production order: this rollout's noise, then this update's permutation
        eps, perm = orc.draw_noise(), orc.draw_perm()
        before = dict(params=named(ac, ac.flat), m=named(ac, alg.optimizer.m), v=named(ac, alg.optimizer.v),
                      hist_m=named(ac, alg.hist_encoder_optimizer.m), hist_v=named(ac, alg.hist_encoder_optimizer.v))
        # this rollout's simulator states (relative to the env origins at its start), with the scheduled terminations
        sims = []
        for t in range(T):
            sim = E.sim_state(p, SEED, step + t + 1, env.env_origins)
            sched.apply(p, sim, step + t + 1)
            for k in SIM_KEYS:
                prod.pool[t][k].copy_(torch.from_numpy(sim[k]))
            sims.append({k: sim[k] for k in SIM_KEYS})
        tables = [env.fill_uniform(step + t + 1).cpu() for t in range(T)]

        env.update_command_curriculum()
        obs = prod.rollout(dagger)
        alg.compute_returns(obs)
        snap = snapshot(prod, sims, tables, precision)
        res = [alg.update_dagger()] if dagger else list(alg.update())
        prod.obs = obs
        step += T
        snap.update(before, result=res, params_after=named(ac, ac.flat))
        S.check(env.common_step_counter == step and s.step == 0, f"iteration {it}: env step {env.common_step_counter}, storage step {s.step}")
        if prev_last_obs is not None:
            S.exact("obs row 0 = the last rollout's obs row T", snap["obs"][0], prev_last_obs)
        prev_last_obs = snap["obs"][T]

        orc.rollout(S, snap, eps, dagger, TOL[precision]["fwd"], sched.resets)
        orc.gae(S, snap)
        if dagger:
            orc.dagger(S, snap, perm)
        else:
            orc.ppo(S, snap, perm)
        S.check(alg.counter == orc.counter, f"iteration {it}: counter {alg.counter}, the reference's {orc.counter}")

    # the Adam step counts: the GPU's own against the reference's per-parameter counts
    S.check(alg.optimizer.step == orc.adam.state["std"]["step"], f"Adam steps {alg.optimizer.step}, the reference's {orc.adam.state['std']['step']}")
    hname = next(n for n in orc.hist_adam.names)
    S.check(alg.hist_encoder_optimizer.step == orc.hist_adam.state[hname]["step"], "history-encoder Adam steps")
    # episodes (OPR:140-154)
    got, want = alg.episode_buffers(), orc.episodes.buffers()
    S.exact("episodes lengths", torch.tensor(got["lenbuffer"]), torch.tensor(want["lenbuffer"]))
    if len(got["rewbuffer"]) == len(want["rewbuffer"]):
        # a return sums `len` rewards, each within FTOL of the oracle's, in fp32 on both sides
        lens = torch.tensor(want["lenbuffer"], dtype=torch.float64)
        for k, rmax in (("rewbuffer", orc.cov["rmax"][0]), ("arm_rewbuffer", orc.cov["rmax"][1])):
            g, w = torch.tensor(got[k], dtype=torch.float64), torch.tensor(want[k], dtype=torch.float64)
            d = (g - w).abs()
            bound = lens * (FTOL["atol"] + FTOL["rtol"] * rmax + 2.4e-7 * w.abs().clamp(min=1.0))
            S.worst[f"episodes {k}"] = float(d.max())
            S.check(bool((d <= bound).all()), f"episodes {k}: {int((d > bound).sum())} returns beyond the bound, max {float(d.max()):.3g}")

    cov = orc.cov
    elapsed = time.perf_counter() - t_start
    print(f"\n[{config} N={N} {precision}{' graphs' if graphs else ''}] worst error per stage: " +
          ", ".join(f"{k} {v:.3g}" for k, v in S.worst.items()))
    print(f"  coverage: time-outs {cov['time_outs']}, terminations {cov['terminations']} ({cov['scheduled']} scheduled), pushes "
          f"{cov['pushes']}, command resamples {cov['resampled']}, clipped ratios {cov['clipped']} of {cov['rows']}, mixing {cov['mixing']}, "
          f"priv-reg {cov['priv_reg']}, finished episodes {len(want['lenbuffer'])}; {elapsed:.1f} s")
    assert not S.failed, "stages that disagree with the oracle:\n  " + "\n  ".join(S.failed)
    # every branch of the join fired
    assert cov["time_outs"] > 0 and cov["terminations"] > 0 and cov["scheduled"] == len(ITERATIONS) * T, cov
    assert cov["pushes"] == 1 and cov["resampled"] > 0 and cov["clipped"] > 0, cov
    assert len(set(cov["lin_vel_x"])) == len(ITERATIONS), cov["lin_vel_x"]
    assert len(set(cov["mixing"])) == 3 and all(0 < x < 1 for x in cov["mixing"][1:]), cov["mixing"]
    assert len(set(cov["priv_reg"])) == 3 and all(0 < x < 1 for x in cov["priv_reg"][1:]), cov["priv_reg"]
    assert len(want["lenbuffer"]) > 0
