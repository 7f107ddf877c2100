"""CUDA-graph capture of a whole rollout for device-resident simulators (the synthetic workload of bench.py and the tests).

`RolloutGraph.run()` captures the T-step sequence of `FusedPPO.act`, `FusedWidowGo1Core.pre_physics_step` and `post_physics_step` once
(per key) and replays it once per iteration.  Every step writes the fixed storage rows of its t (observations t + 1, rewards / dones t),
so the captured pointers stay valid; the values that change between replays are drawn or copied eagerly before the replay:
  * the standard normals of the whole rollout, by the same generator call as the eager path (`FusedPPO.act` at t = 0);
  * the step record of the post-physics kernel (step, push interval, curriculum values): one asynchronous stream-ordered copy.  The kernel reads it
    and the step advances on the device after each use, so two replays continue the Philox stream exactly as two eager rollouts do.
Per-step statistics are not read on the host (sync_stats=False semantics); `env.episode_stats()` reads the device accumulators once
per iteration.  The Isaac Gym drop-in is not captured: its physics calls run between the segments of each env step.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L


class HostUpload:
    """Host values into a device buffer with one asynchronous, stream-ordered copy: the values go through a pinned staging buffer, which
    is refilled only after the copy that last read it has run (a pageable source would make the copy wait for the whole stream)."""

    def __init__(self):
        self._pinned, self._done = None, None

    def __call__(self, dst: torch.Tensor, host: torch.Tensor):
        if self._pinned is None or self._pinned.shape != host.shape or self._pinned.dtype != host.dtype:
            self._pinned, self._done = torch.empty(host.shape, dtype=host.dtype).pin_memory(), None
        if self._done is not None:
            self._done.synchronize()
        self._pinned.copy_(host)
        dst.copy_(self._pinned, non_blocking=True)
        self._done = torch.cuda.Event()
        self._done.record()


# DwbcEnvBuffers fields a captured rollout sets per step itself (observation / transition targets) or re-binds through physics(t)
_PER_STEP_FIELDS = {"obs_buf", "obs_stride", "store_values", "store_rewards", "store_dones", "store_gamma", "reserved_", "root_states",
                    "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques"}


class RolloutGraph:
    def __init__(self, alg, env, physics=None):
        """`physics(t)` stands for the simulator of step t.  It runs during capture only: it may re-bind the core's simulator tensors
        (`env.bind_sim`) or enqueue device work, and must not read results on the host.  The simulator tensors it binds are part of the
        graph: binding other tensors at run time needs a new RolloutGraph."""
        self.alg, self.env, self.physics = alg, env, physics
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
        T, n = s.num_transitions_per_env, s.num_envs
        na = alg.actor_critic.num_leg_actions + alg.actor_critic.num_arm_actions
        if alg._eps_all is None or alg._eps_all.shape[:2] != (T, n):
            alg._eps_all = torch.empty(T, n, na, device=alg.device)
            alg._eps_valid = False
        alg._workspace(n)
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
        alg._workspace(s.num_envs)
        key = self.key(hist_encoding)
        if key not in self._graphs:
            self._capture(key, hist_encoding)
        row0 = s.obs_row(0)
        if obs.data_ptr() != row0.data_ptr():
            row0.copy_(obs)
        alg._eps_all.normal_(generator=alg.generator)                                   # FusedPPO.act at t = 0
        alg._eps_valid = True
        self._upload(self._record, env.step_record())
        self._graphs[key].replay()
        T = s.num_transitions_per_env
        s.step = T
        env.common_step_counter += T
        alg._packed, alg._packed_key = True, (s.num_envs, int(bool(hist_encoding)), alg.actor_critic.flat._version)
        env.set_obs_target(s.obs_row(T))
        env.extras["time_outs"] = env.time_out_buf
        env.extras["dwbc_stored_rows"] = (s.rewards[T - 1].data_ptr(), s.dones[T - 1].data_ptr())
        return env.obs_buf
