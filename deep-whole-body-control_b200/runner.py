"""`OnPolicyRunner.learn` (rsl_rl/rsl_rl/runners/on_policy_runner.py:100-177, cited OPR:line) for device-resident simulators, with the
host reading results once per log interval instead of once per step.

`GraphRunner.learn()` runs OPR.learn's iterations in its order: the command curriculum, the teacher / student choice (OPR:129), the
rollout (a `RolloutGraph`), `compute_returns`, `update()` or `update_dagger()` (OPR:166-169) and the checkpoint cadence (OPR:175-176).
Nothing in that loop needs a device result on the host: the schedules and the curriculum are host arithmetic on iteration counts, and
the noise and the permutation come from the generator.  So the iterations are enqueued ahead of the GPU, and each one ends with
stream-ordered device-to-device copies of what OPR.log reports (the loss sums, std, the episode tracker, the env's episode statistics,
the update diagnostics) into a ring of `log_interval` rows.  `logs()` reads the ring with one synchronisation and applies the host
arithmetic of FusedPPO's and the env's own readers to it, so every value is bitwise what an eager loop reading every iteration gets
(DESIGN §14).  The Isaac Gym drop-in is not covered: its physics runs as host calls between the segments of every env step.

With `eval_env`, the deterministic teacher and / or student (EvalGraph) are evaluated on a core of their own every `eval_interval`
iterations, each run from the same snapshot of that core, and their episode results join the iteration's row by the same device copies.
With `timing=True`, CUDA events on the stream give each row OPR.log's collection / learning times and fps in GPU time.
"""
from __future__ import annotations

import statistics

import numpy as np
import torch

from . import _lib as L
from .graphs import EvalGraph, RolloutGraph
from .ppo import dagger_loss, diagnostics_from, loss_means, ppo_result, ring_buffers

# update()'s 7-tuple under the names OPR.learn gives it (OPR:169), and what a DAgger iteration reports instead (OPR:167)
PPO_KEYS = ("mean_value_loss", "mean_surrogate_loss", "mean_arm_torques_loss", "mean_value_mixing_ratio",
            "mean_torque_supervision_weight", "mean_priv_reg_loss", "priv_reg_coef")
DAGGER_KEY = "mean_hist_latent_loss"
# OPR.log's means over the tracker's deques (None while no episode has finished), by deque
EPISODE_MEANS = (("rewbuffer", "mean_reward"), ("arm_rewbuffer", "mean_arm_reward"), ("lenbuffer", "mean_episode_length"))
# the policies a scheduled evaluation can run, in the order they run: the actor alone, and the actor with the history-encoder latent
EVAL_MODES = ("teacher", "student")
# the row values timing=True adds; GPU times are not bitwise, so comparisons of rows leave these out
TIMING_KEYS = ("collection_time", "learn_time", "fps", "tot_timesteps", "tot_time", "learning_rate", "eval_time", "captured")


def _positive_int(name, v):
    if isinstance(v, bool) or not isinstance(v, int) or v <= 0:
        raise L.DwbcError(f"{name} must be a positive int, not {v!r}")
    return v


def _plain(x):
    """Numpy scalars (the curriculum coefficients of extras['episode']) as Python floats, so that a checkpoint loads with
    torch.load(weights_only=True)."""
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, list):
        return [_plain(v) for v in x]
    return float(x) if isinstance(x, np.generic) else x


class GraphRunner:
    _Event = torch.cuda.Event               # the timing events (a test substitutes host clocks)

    def __init__(self, alg, env, physics=None, log_interval=10, save_interval=500, save_path=None, capture=False, eval_env=None,
                 eval_interval=None, eval_steps=None, eval_track_episodes=100, eval_physics=None, eval_modes=EVAL_MODES, timing=False):
        """`alg`: a FusedPPO with storage and an episode tracker (track_episodes=C > 0: the mean reward and episode length are the first
        things OPR.log prints); `env`: a FusedWidowGo1Core with sync_stats=False; `physics(t)` as for RolloutGraph.  `log_interval`: the
        rows of the device log ring, i.e. how many iterations are enqueued before the host reads (logs() reads earlier).
        `save_path(it)`: the checkpoint file after iteration `it` when it % save_interval == 0 and after the last one (OPR:175-176,
        the file names of OPR.save); None saves nothing.  `capture=False` issues the launches of the captured rollout and update
        eagerly, with the same bits.

        `eval_env`: a second FusedWidowGo1Core (sync_stats=False) on which, after the update of each iteration `it` with
        it % eval_interval == 0, every mode of `eval_modes` runs an EvalGraph of `eval_steps` steps (even) with a tracker of
        `eval_track_episodes` episodes and `eval_physics(t)` as its simulator.  Its state_dict() is taken here, with the curriculum and
        episode lengths the caller set, and restored before each mode's run, so every evaluation starts from the same task state.
        `timing=True`: each row gains OPR.log's throughput figures, from CUDA events on the current stream."""
        self.alg, self.env, self.physics = alg, env, physics
        self.log_interval = _positive_int("log_interval", log_interval)
        self.save_interval = _positive_int("save_interval", save_interval)
        self.save_path, self.capture = save_path, bool(capture)
        self.eval_env, self._evals = eval_env, {}
        if eval_env is not None:
            if eval_env is env:
                raise L.DwbcError("an evaluation moves the core it runs on: give eval_env a core of its own, not the training core")
            self.eval_interval = _positive_int("eval_interval", eval_interval)
            if isinstance(eval_modes, str) or not set(eval_modes) <= set(EVAL_MODES) or not eval_modes:
                raise L.DwbcError(f"eval_modes must be a non-empty subset of {EVAL_MODES}, not {eval_modes!r}")
        self._check()
        if eval_env is not None:
            self._evals = {m: EvalGraph(alg.actor_critic, eval_env, eval_steps, hist_encoding=m == "student",
                                        track_episodes=eval_track_episodes, physics=eval_physics, capture=self.capture)
                           for m in EVAL_MODES if m in eval_modes}
            self._eval_start = eval_env.state_dict()
        self.rollout = RolloutGraph(alg, env, physics, capture=self.capture)
        self.current_learning_iteration = 0
        n, dev = self.log_interval, alg.device
        z = lambda *s, dtype=torch.float32: torch.zeros(n, *s, dtype=dtype, device=dev)  # noqa: E731
        ep = alg._episodes
        self._ring = dict(losses=z(*alg._losses.shape), std=z(alg.actor_critic.std.numel()), ring=z(*ep["ring"].shape),
                          pos=z(*ep["pos"].shape, dtype=ep["pos"].dtype), stats=z(*env._stats.shape))
        if alg.diagnostics:
            self._ring.update(diag=z(*alg._diag_buffer().shape), ev=z(*alg._diag_ev.shape))
        for m, ev in self._evals.items():
            e = ev._episodes
            self._ring.update({f"eval.{m}.ring": z(*e["ring"].shape), f"eval.{m}.pos": z(*e["pos"].shape, dtype=e["pos"].dtype),
                               f"eval.{m}.stats": z(*eval_env._stats.shape)})
        # per row: before the rollout, after it, after the update, before and after the evaluation
        self._events = [[self._Event(enable_timing=True) for _ in range(5)] for _ in range(n)] if timing else None
        self.tot_timesteps, self.tot_time = 0, 0.0        # OPR's totals over this runner's logged iterations
        self._host = []              # the host-side values of each row enqueued in the ring, oldest first
        self._rows = []              # rows read from the ring that logs() has not returned yet

    def _check(self):
        """The refusals, before any launch."""
        alg, env = self.alg, self.env
        if alg.world_size > 1:
            raise L.DwbcError("GraphRunner runs one GPU: world_size must be 1")
        if env.sync_stats or (self.eval_env is not None and self.eval_env.sync_stats):
            raise L.DwbcError("GraphRunner reads no per-step statistics: build the env cores with sync_stats=False")
        if alg.storage is None:
            raise L.DwbcError("GraphRunner needs a FusedPPO with storage: call alg.init_storage() first")
        if alg.storage.step != 0:
            raise L.DwbcError(f"the storage holds {alg.storage.step} steps of a rollout: GraphRunner starts between iterations")
        if not alg.track_episodes:
            raise L.DwbcError("GraphRunner logs the mean reward and episode length: use FusedPPO(track_episodes=C > 0)")

    @staticmethod
    def dagger_iteration(it, dagger_update_freq):
        """OPR:129: the student (history encoder) acts, and update_dagger() replaces update(), on these iterations."""
        return it % dagger_update_freq == 0

    def learn(self, num_learning_iterations, init_at_random_ep_len=False):
        """OPR.learn's iterations current_learning_iteration .. + num_learning_iterations - 1, enqueued without waiting for the GPU.
        The host reads only to save a checkpoint and when the log ring is full; the first run of each rollout key, update kind and
        evaluation mode captures its graph (capture=True), which synchronises once."""
        self._check()
        env, alg = self.env, self.alg
        if init_at_random_ep_len:
            env.episode_length_buf = torch.randint_like(env.episode_length_buf, high=int(env.max_episode_length))     # OPR:107-108
        obs = env.get_observations()
        start = self.current_learning_iteration
        for it in range(start, start + num_learning_iterations):
            if len(self._host) == self.log_interval:
                self._read()
            events = None if self._events is None else self._events[len(self._host)]
            graphs = None if events is None else self._graphs()
            env.update_command_curriculum()
            hist_encoding = self.dagger_iteration(it, alg.dagger_update_freq)
            self._record(events, 0)
            obs = self.rollout.run(obs, hist_encoding)
            self._record(events, 1)
            alg.compute_returns(obs)
            if hist_encoding:
                alg._dagger_run(self.capture)
                alg._dagger_end()
                sched = None
            else:
                sched = alg._ppo_end(alg._ppo_run(self.capture))
            self._record(events, 2)
            self._snapshot(it, sched)
            if self._evals and it % self.eval_interval == 0:
                self._record(events, 3)
                self._evaluate()
                self._record(events, 4)
            if events is not None:
                s = alg.storage
                self._host[-1].update(steps=s.num_transitions_per_env * s.num_envs, learning_rate=alg.learning_rate,
                                      captured=[id(g) for g in self._graphs()] != [id(g) for g in graphs])
            self.current_learning_iteration = it + 1
            if self.save_path is not None and it % self.save_interval == 0:
                self.save(self.save_path(it))
        if self.save_path is not None:
            self.save(self.save_path(self.current_learning_iteration))

    @staticmethod
    def _record(events, i):
        if events is not None:
            events[i].record()

    def _graphs(self):
        """Every captured graph object; a list that differs after an iteration means the iteration captured one."""
        return (list(self.rollout._graphs.values()) + [g["graph"] for g in self.alg._graphs.values()] +
                [ev._graph for ev in self._evals.values()])

    def _snapshot(self, it, sched):
        """Enqueue this iteration's log row: device-to-device copies into the ring, then the env's episode statistics are reset on the
        device as episode_stats() resets them.  `sched`: _ppo_end's schedule values, None on a DAgger iteration."""
        if len(self._host) == self.log_interval:
            self._read()
        k, r, alg, env = len(self._host), self._ring, self.alg, self.env
        r["losses"][k].copy_(alg._losses)
        r["std"][k].copy_(alg.actor_critic.std.reshape(-1))
        r["ring"][k].copy_(alg._episodes["ring"])
        r["pos"][k].copy_(alg._episodes["pos"])
        r["stats"][k].copy_(env._stats)
        env._stats.zero_()
        if sched is not None and alg.diagnostics:
            r["diag"][k].copy_(alg._diag)
            r["ev"][k].copy_(alg._diag_ev)
        self._host.append(dict(iteration=it, sched=sched, coeffs=env._curriculum_coeffs(), eval_coeffs=None))

    def _evaluate(self):
        """Enqueue an evaluation of each mode into the newest row: the eval core restored to the snapshot (in-place copies, so the
        captured evaluation stays valid), the mode's tracker zeroed, its EvalGraph run, and the tracker and the core's episode
        statistics copied into the ring; the statistics are then reset on the device, as EvalGraph.results() resets them."""
        k, r, env = len(self._host) - 1, self._ring, self.eval_env
        for m, ev in self._evals.items():
            env.load_state_dict(self._eval_start)
            for v in ev._episodes.values():
                v.zero_()
            ev.run(env.obs_buf)
            r[f"eval.{m}.ring"][k].copy_(ev._episodes["ring"])
            r[f"eval.{m}.pos"][k].copy_(ev._episodes["pos"])
            r[f"eval.{m}.stats"][k].copy_(env._stats)
            env._stats.zero_()                       # as results() leaves it
        self._host[-1]["eval_coeffs"] = env._curriculum_coeffs()

    def _read(self):
        """Read the enqueued rows with one synchronisation and turn them into log rows."""
        if not self._host:
            return
        alg, env, n = self.alg, self.env, len(self._host)
        num_updates = alg.num_learning_epochs * alg.num_mini_batches
        dev = dict(self._ring, means=loss_means(self._ring["losses"], num_updates))
        host = {k: v[:n].to("cpu", non_blocking=True) for k, v in dev.items()}
        if alg.device.type == "cuda":
            torch.cuda.current_stream(alg.device).synchronize()
        for i, h in enumerate(self._host):
            row = dict(iteration=h["iteration"], hist_encoding=h["sched"] is None)
            if h["sched"] is None:
                row[DAGGER_KEY] = dagger_loss(host["losses"][i, 0], num_updates)
            else:
                losses = host["means"][i].tolist()
                alg.last_entropy = losses[3]
                row.update(zip(PPO_KEYS, ppo_result(losses, h["sched"], alg.torque_supervision)))
            bufs = ring_buffers(host["ring"][i], host["pos"][i])
            for buf, key in EPISODE_MEANS:
                row[key] = statistics.mean(bufs[buf]) if bufs[buf] else None        # OPR.log
            env._fill_episode_extras(host["stats"][i], h["coeffs"])
            row["episode"] = dict(env.extras["episode"])
            row["std"] = host["std"][i].tolist()
            if alg.diagnostics:
                row["diagnostics"] = None if h["sched"] is None else diagnostics_from(host["diag"][i], host["ev"][i])
            if self._evals:
                row["eval"] = None if h["eval_coeffs"] is None else {m: self._eval_row(host, i, m, h["eval_coeffs"]) for m in self._evals}
            if self._events is not None:
                row.update(self._timing(self._events[i], h))
            self._rows.append(row)
        self._host = []

    def _eval_row(self, host, i, m, coeffs):
        """One mode's results in row i, as EvalGraph.results() and OPR.log give them: the means over the tracker's last C episodes
        (None when none finished), the number of episodes finished and the eval core's extras['episode']."""
        pos = host[f"eval.{m}.pos"][i]
        bufs = ring_buffers(host[f"eval.{m}.ring"][i], pos)
        out = {key: statistics.mean(bufs[buf]) if bufs[buf] else None for buf, key in EPISODE_MEANS}
        out["num_episodes"] = int(pos[1])
        self.eval_env._fill_episode_extras(host[f"eval.{m}.stats"][i], coeffs)
        out["episode"] = dict(self.eval_env.extras["episode"])
        return out

    def _timing(self, events, h):
        """OPR.log's throughput figures (OPR:128, 156-157, 171-172, 206) from the row's events, in GPU seconds; compute_returns counts
        as learning.  A row whose iteration captured a graph includes the host's capture time (`captured`)."""
        collection, learn = events[0].elapsed_time(events[1]) / 1e3, events[1].elapsed_time(events[2]) / 1e3
        self.tot_timesteps += h["steps"]
        self.tot_time += collection + learn
        out = dict(collection_time=collection, learn_time=learn, fps=int(h["steps"] / (collection + learn)),
                   tot_timesteps=self.tot_timesteps, tot_time=self.tot_time, learning_rate=h["learning_rate"], captured=h["captured"])
        if h["eval_coeffs"] is not None:
            out["eval_time"] = events[3].elapsed_time(events[4]) / 1e3
        return out

    def logs(self):
        """One dict per iteration since the last call, oldest first, read with one synchronisation: `iteration`, `hist_encoding`, the
        update's results (PPO_KEYS, or DAGGER_KEY on a DAgger iteration), OPR.log's `mean_reward`, `mean_arm_reward` and
        `mean_episode_length` (None while no episode has finished), `episode` (env.episode_stats() of the iteration), the policy's
        `std` after the update and, with FusedPPO(diagnostics=True), `diagnostics` (update_diagnostics(); None on DAgger iterations).
        With eval_env, `eval`: None, or on evaluated iterations {mode: {mean_reward, mean_arm_reward, mean_episode_length (None when no
        episode finished), num_episodes, episode}}.  With timing=True, TIMING_KEYS: `collection_time` and `learn_time` (GPU seconds),
        `fps`, `tot_timesteps` and `tot_time` (since this runner was built), `learning_rate`, `captured`, and `eval_time` on evaluated
        iterations.  Sets alg.last_entropy as update() does."""
        self._read()
        rows, self._rows = self._rows, []
        return rows

    def save(self, path, infos=None):
        """OPR.save's checkpoint (OPR:276-282: model_state_dict, optimizer_state_dict, iter, infos; `iter` is the next iteration), and
        under 'dwbc' what load() needs to continue bit for bit: alg.state_dict(), env.state_dict(), the iteration and the log rows not
        yet returned by logs(); with eval_env also 'eval': the eval core's start snapshot and its carried extras['episode'].  The
        simulator's own state is the caller's (DESIGN §10)."""
        self._read()
        alg, it = self.alg, self.current_learning_iteration
        dwbc = dict(alg=alg.state_dict(), env=self.env.state_dict(), iteration=it, logs=_plain(self._rows),
                    episode=_plain(dict(self.env.extras["episode"])))
        if self._evals:
            dwbc["eval"] = dict(start=self._eval_start, episode=_plain(dict(self.eval_env.extras["episode"])))
        torch.save(dict(model_state_dict=alg.actor_critic.state_dict(), optimizer_state_dict=alg.optimizer.state_dict(), iter=it,
                        infos=infos, dwbc=dwbc), path)

    def load(self, path):
        """Restore a save(): the training state, the iteration, the unread log rows, the episode values extras['episode'] carries
        over iterations in which no episode ends and, with eval_env, the evaluations' start snapshot.  A checkpoint with an
        evaluation snapshot needs a runner with eval_env, and the reverse.  Returns the checkpoint's `infos`."""
        ck = torch.load(path, weights_only=True)
        d = ck.get("dwbc") if isinstance(ck, dict) else None
        if not isinstance(d, dict) or set(d) - {"eval"} != {"alg", "env", "iteration", "logs", "episode"}:
            raise L.DwbcError(f"{path} is not a GraphRunner checkpoint")
        if ("eval" in d) != bool(self._evals):
            raise L.DwbcError(f"{path} {'holds' if 'eval' in d else 'holds no'} evaluation snapshot, and this runner "
                              f"{'evaluates' if self._evals else 'does not evaluate'}: build it with{'' if 'eval' in d else 'out'} eval_env")
        if self._evals:
            self.eval_env.load_state_dict(d["eval"]["start"])       # refuses a snapshot of another core before the training state moves
        self.alg.load_state_dict(d["alg"])
        self.env.load_state_dict(d["env"])
        self.current_learning_iteration = int(d["iteration"])
        self._host, self._rows = [], list(d["logs"])
        self.env.extras["episode"] = dict(d["episode"])
        if self._evals:
            self._eval_start = d["eval"]["start"]
            self.eval_env.extras["episode"] = dict(d["eval"]["episode"])
        return ck.get("infos")
