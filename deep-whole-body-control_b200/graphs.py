"""CUDA-graph capture of a whole rollout for device-resident simulators (the synthetic workload of bench.py and the tests).

`RolloutGraph.run()` captures the T-step sequence of `FusedPPO.act`, `FusedWidowGo1Core.pre_physics_step` and `post_physics_step` once
(per key) and replays it once per iteration.  Every step writes the fixed storage rows of its t (observations t + 1, rewards / dones t),
so the captured pointers stay valid; the values that change between replays are drawn or copied eagerly before the replay:
  * the standard normals of the whole rollout, by the same generator call as the eager path (`FusedPPO.act` at t = 0);
  * the step record of the post-physics kernel (step, push interval, curriculum values): one asynchronous stream-ordered copy.  The kernel reads it
    and the step advances on the device after each use, so two replays continue the Philox stream exactly as two eager rollouts do.
Per-step statistics are not read on the host (sync_stats=False semantics); `env.episode_stats()` reads the device accumulators once
per iteration.  The Isaac Gym drop-in is not captured: its physics calls run between the segments of each env step.

`EvalGraph.run()` captures a deterministic evaluation rollout the same way, with no training state: the action mean of the actor alone
(dwbc_policy_mean), the env step, and the runner's episode bookkeeping (dwbc_track_episodes) into a tracker of its own.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L
from .actor_critic import PolicyMean


class HostUpload:
    """Host values into a device buffer with one asynchronous, stream-ordered copy that never waits for the device.  The values go
    through a fresh pinned staging buffer from PyTorch's caching host allocator, which records the copy and hands the buffer out again
    only once the copy has run (a pageable source would make the copy wait for the whole stream, and refilling one staging buffer would
    wait for the copy before).  So a loop can enqueue many iterations ahead of the GPU (GraphRunner)."""

    def __call__(self, dst: torch.Tensor, host: torch.Tensor):
        dst.copy_(host.pin_memory(), non_blocking=True)


# DwbcEnvBuffers fields a captured rollout sets per step itself (observation / transition targets) or re-binds through physics(t)
_PER_STEP_FIELDS = {"obs_buf", "obs_stride", "store_values", "store_rewards", "store_dones", "store_gamma", "reserved_", "root_states",
                    "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques"}


class RolloutGraph:
    def __init__(self, alg, env, physics=None, capture=True):
        """`physics(t)` stands for the simulator of step t.  It runs during capture only: it may re-bind the core's simulator tensors
        (`env.bind_sim`) or enqueue device work, and must not read results on the host.  The simulator tensors it binds are part of the
        graph: binding other tensors at run time needs a new RolloutGraph.  `capture=False` issues the same launches eagerly on every
        run, physics(t) included."""
        self.alg, self.env, self.physics, self.capture = alg, env, physics, bool(capture)
        self._graphs = {}                        # key() -> CUDAGraph: PPO and DAgger rollouts alternate without re-capturing
        self._record = torch.zeros(C.sizeof(L.StepDevice), dtype=torch.uint8, device=env.device)
        self._upload = HostUpload()

    def key(self, hist_encoding):
        """What a captured rollout depends on: the history-encoder flag, the policy (precision, network, parameters, workspace), the
        storage, the env core's configuration and task-state buffers (a new tensor bound there, e.g. by `load_state`, re-captures), and
        the episode tracker's buffers when FusedPPO(track_episodes=C > 0)."""
        a, s, e = self.alg, self.alg.storage, self.env
        env_bufs = tuple(getattr(e._buf, f) for f, _ in L.EnvBuffers._fields_ if f not in _PER_STEP_FIELDS)
        tracker = () if a._episodes is None else ((a.track_episodes,) + tuple(v.data_ptr() for v in a._episodes.values()),)
        return (bool(hist_encoding), a.precision, s.num_transitions_per_env, s.num_envs, s._obs_all.data_ptr(), a._ws.data_ptr(),
                a._ws_rows, a.actor_critic.flat.data_ptr(), bytes(a.actor_critic.net_cfg), a.gamma, bytes(e._cfg), env_bufs,
                int(e._args.generic_kernel), e.seed) + tracker

    def _steps(self, hist_encoding):
        """The launches of one rollout, exactly as an eager loop issues them (bench.Workload.rollout)."""
        alg, env, s = self.alg, self.env, self.alg.storage
        obs = s.obs_row(0)
        for t in range(s.num_transitions_per_env):
            actions = alg.act(obs, obs, hist_encoding, eps=alg._eps_all[t])
            if self.physics is not None:
                self.physics(t)
            env.set_obs_target(s.obs_row(t + 1))
            env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
            env.pre_physics_step(actions)
            env.post_physics_step()
            obs = env.obs_buf
            alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
        return obs

    def _capture(self, key, hist_encoding):
        alg, env, s = self.alg, self.env, self.alg.storage
        self._graphs.pop(key, None)
        counter = env.common_step_counter
        alg._packed = False                          # step 0 of every replay packs the weight images, as the first eager act() does
        env.set_device_step(self._record)
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(env.device)
        try:
            with torch.cuda.graph(graph):
                self._steps(hist_encoding)
        finally:
            env.common_step_counter = counter      # capture ran no step
            s.step = 0
            env.set_device_step(None)
        self._graphs[key] = graph

    def run(self, obs, hist_encoding=False):
        """One rollout into the storage rows: obs_0 -> row 0 (copied unless it is row 0 already), returns obs_T (row T)."""
        alg, env, s = self.alg, self.env, self.alg.storage
        if env.sync_stats:
            raise L.DwbcError("a captured rollout reads no per-step statistics: use sync_stats=False and env.episode_stats()")
        if s.step != 0:
            raise L.DwbcError("a captured rollout starts at storage row 0")
        alg._set_precision()
        T, n = s.num_transitions_per_env, s.num_envs
        alg._workspace(n)
        na = alg.actor_critic.num_leg_actions + alg.actor_critic.num_arm_actions
        if alg._eps_all is None or alg._eps_all.shape[:2] != (T, n):
            alg._eps_all = torch.empty(T, n, na, device=alg.device)
            alg._eps_valid = False
        if self.capture:
            key = self.key(hist_encoding)
            if key not in self._graphs:
                self._capture(key, hist_encoding)
        row0 = s.obs_row(0)
        if obs.data_ptr() != row0.data_ptr():
            row0.copy_(obs)
        alg._eps_all.normal_(generator=alg.generator)                                   # FusedPPO.act at t = 0
        alg._eps_valid = True
        if not self.capture:
            return self._steps(hist_encoding)
        self._upload(self._record, env.step_record())
        self._graphs[key].replay()
        s.step = T
        env.common_step_counter += T
        alg._packed, alg._packed_key = True, (s.num_envs, int(bool(hist_encoding)), alg.actor_critic.flat._version)
        env.set_obs_target(s.obs_row(T))
        env.extras["time_outs"] = env.time_out_buf
        env.extras["dwbc_stored_rows"] = (s.rewards[T - 1].data_ptr(), s.dones[T - 1].data_ptr())
        return env.obs_buf


class EvalGraph:
    """A deterministic evaluation of `policy` (FlatActorCritic or FusedActorCritic) on the device-resident `env` core over `steps` env
    steps, captured as one CUDA graph (capture=False: the same launches, eager).  Each step: the action mean (dwbc_policy_mean, the
    precision in the policy's net_cfg), env.pre_physics_step(mean), physics(t), env.post_physics_step(), dwbc_track_episodes on the
    un-bootstrapped rewards and dones.  No noise is drawn and nothing is stored.  The observations ping-pong between two fixed rows (step t
    reads row t % 2 and writes row (t + 1) % 2), so `steps` is even and obs_T is row 0.  The step record goes up once per run (HostUpload)
    and advances on the device, so the env's Philox stream and common_step_counter continue across runs as eager steps do.

    `env` should be a core of its own: the evaluation moves its state, and its transition target is switched off.  `physics(t)` as for
    RolloutGraph.  `load_state_dict` into the policy between runs is replayed without re-capture (the weight images are rebuilt at step 0
    of every run); any other change in key() re-captures."""

    def __init__(self, policy, env, steps, hist_encoding=False, track_episodes=100, physics=None, capture=True):
        ac = self._core(policy)
        if isinstance(track_episodes, bool) or not isinstance(track_episodes, int) or track_episodes <= 0:
            raise L.DwbcError(f"track_episodes must be a positive int (the number of finished episodes kept), not {track_episodes!r}")
        if isinstance(steps, bool) or not isinstance(steps, int) or steps <= 0 or steps % 2:
            raise L.DwbcError(f"steps must be a positive even int (the observations ping-pong between two rows), not {steps!r}")
        na = ac.num_leg_actions + ac.num_arm_actions
        if ac.num_obs != env.num_obs or na != env.num_actions:
            raise L.DwbcError(f"the policy takes {ac.num_obs} observations and gives {na} actions, the env core {env.num_obs} and "
                              f"{env.num_actions}")
        self.policy, self.env, self.steps, self.hist_encoding = policy, env, steps, bool(hist_encoding)
        self.track_episodes, self.physics, self.capture = track_episodes, physics, bool(capture)
        N, dev = env.num_envs, env.device
        self._obs = torch.zeros(2, N, (env.num_obs + 3) // 4 * 4, device=dev)        # rows start 16-byte aligned (set_obs_target)
        self._actions = torch.zeros(N, na, device=dev)
        self._mean = PolicyMean()
        self._episodes = dict(running=torch.zeros(N, 3, device=dev), ring=torch.zeros(track_episodes, 3, device=dev),
                              pos=torch.zeros(2, dtype=torch.int64, device=dev))
        self._record = torch.zeros(C.sizeof(L.StepDevice), dtype=torch.uint8, device=dev)
        self._upload = HostUpload()
        self._graph = None                       # (key, CUDAGraph)

    @staticmethod
    def _core(policy):
        return getattr(policy, "core", policy)  # FusedActorCritic -> its FlatActorCritic

    def obs_row(self, t):
        """The observation buffer step t reads ([N, >= num_obs]; the columns past num_obs are padding)."""
        return self._obs[t % 2]

    def key(self):
        """What a captured evaluation depends on: the policy (parameter buffer, network, precision), the env core's configuration and
        task-state buffers, the history-encoder flag, the step count and the tracker.  Not the parameter values."""
        ac, e = self._core(self.policy), self.env
        env_bufs = tuple(getattr(e._buf, f) for f, _ in L.EnvBuffers._fields_ if f not in _PER_STEP_FIELDS)
        return (ac.flat.data_ptr(), bytes(ac.net_cfg), bytes(e._cfg), env_bufs, int(e._args.generic_kernel), e.seed, self.hist_encoding,
                self.steps, self.track_episodes, self._mean.reserve(ac, e.num_envs).data_ptr())

    def _steps(self):
        ac, env, e = self._core(self.policy), self.env, self._episodes
        lib = L.lib()
        env.set_transition_target(None)
        for t in range(self.steps):
            self._mean(ac, self.obs_row(t), self._actions, self.hist_encoding, repack=t == 0)
            env.pre_physics_step(self._actions)
            if self.physics is not None:
                self.physics(t)
            env.set_obs_target(self._obs[(t + 1) % 2])
            env.post_physics_step()
            L.check(lib.dwbc_track_episodes(L.ptr(env.rew_buf, torch.float32), L.ptr(env.arm_rew_buf, torch.float32),
                                            L.ptr(env.reset_buf, (torch.uint8, torch.bool)), env.num_envs, L.ptr(e["running"]), L.ptr(e["ring"]),
                                            L.ptr(e["pos"]), self.track_episodes, L.stream_ptr()), "dwbc_track_episodes")

    def _capture(self, key):
        env = self.env
        self._graph = None
        counter = env.common_step_counter
        env.set_device_step(self._record)
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(env.device)
        try:
            with torch.cuda.graph(graph):
                self._steps()
        finally:
            env.common_step_counter = counter      # capture ran no step
            env.set_device_step(None)
        self._graph = (key, graph)

    def run(self, obs):
        """`steps` env steps from obs_0 ([N, >= num_obs], copied unless it is obs_row(0) already); returns obs_T (obs_row(0))."""
        env = self.env
        if env.sync_stats:
            raise L.DwbcError("a captured evaluation reads no per-step statistics: use sync_stats=False and results()")
        row0 = self.obs_row(0)
        if obs.data_ptr() != row0.data_ptr():
            row0[:, :env.num_obs].copy_(obs[:, :env.num_obs])
        if not self.capture:
            self._steps()
        else:
            key = self.key()
            if self._graph is None or self._graph[0] != key:
                self._capture(key)
            self._upload(self._record, env.step_record())
            self._graph[1].replay()
            env.common_step_counter += self.steps
            env.set_obs_target(self._obs[0])
            env.extras["time_outs"] = env.time_out_buf
            env.extras["dwbc_stored_rows"] = None
        return row0

    def results(self, reset=True):
        """OPR's rewbuffer, arm_rewbuffer and lenbuffer (Python float lists, oldest first) of the last track_episodes episodes finished
        in this evaluation's runs, and env.episode_stats(reset) -- read with one synchronisation."""
        ring = self._episodes["ring"].to("cpu", non_blocking=True)
        pos = self._episodes["pos"].to("cpu", non_blocking=True)
        stats = self.env.episode_stats(reset)           # its blocking read orders behind the two copies on the stream
        cap = self.track_episodes
        n = min(int(pos[1]), cap)
        rows = ring[(int(pos[0]) - n + torch.arange(n)) % cap]
        return dict(rewbuffer=rows[:, 0].tolist(), arm_rewbuffer=rows[:, 1].tolist(), lenbuffer=rows[:, 2].tolist(), episode=stats)
