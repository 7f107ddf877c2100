"""TEST INFRASTRUCTURE ONLY -- one full PPO iteration of the hot path on the CPU oracle.

rollout (policy forward -> post-physics step -> reward bootstrap) x T, GAE, update(): the same
sequence `OnPolicyRunner.learn` drives (rsl_rl/rsl_rl/runners/on_policy_runner.py:125-169), on
synthetic sim-state tensors.  Used only by bench.py (`cpu_baseline` leg and `--impl reference`:
the reference is pure Python and may not be installed where the benchmark runs, so the pinned
oracle port is what runs there).  The tests check the production loop stage by stage instead
(tests/test_gpu_training_iteration.py), each stage recomputed from the GPU's previous one.
"""
from __future__ import annotations

import time
from types import SimpleNamespace

import numpy as np
import torch

from . import env_oracle as EO, ppo_oracle as PO


class OracleIteration:
    def __init__(self, p, init_state, runtime, params, hp, sim_fn, rand_fn, T):
        """p: task params; init_state: oracle SimpleNamespace; sim_fn(t)->dict of numpy sim tensors;
        rand_fn(t)->uniform table."""
        self.p, self.rt, self.P, self.hp, self.T = p, runtime, params, hp, T
        self.env = EO.EnvOracle(p, init_state)
        self.sim_fn, self.rand_fn = sim_fn, rand_fn
        self.opt = PO.Adam(list(params.keys()), hp["learning_rate"])
        self.counter = 1500
        self.N = p.num_envs
        self.obs = torch.zeros(self.N, p.num_obs)
        self.step_count = 0

    def _load(self, sim, actions):
        s, p = self.env.s, self.p
        s.root_states_full.copy_(torch.from_numpy(sim["root_states"]))
        s.dof_state.copy_(torch.from_numpy(sim["dof_state"]))
        s.rigid_body_state.copy_(torch.from_numpy(sim["rigid_body_state"]))
        s.contact_forces_full.copy_(torch.from_numpy(sim["contact_forces"]))
        s.force_sensor.copy_(torch.from_numpy(sim["force_sensor"]))
        s.torques = torch.from_numpy(sim["torques"]).clone()
        a = torch.clip(actions[:, p.raisim2ig(p.num_actions)], -100.0, 100.0)
        s.action_history_buf = torch.cat([s.action_history_buf[:, 1:], a[:, None, :]], dim=1)
        s.actions = s.action_history_buf[:, -3].clone()

    def run(self):
        """One iteration; returns dict of timings (s) for rollout / gae / update."""
        p, T, N, hp = self.p, self.T, self.N, self.hp
        st = dict(observations=torch.zeros(T, N, p.num_obs), actions=torch.zeros(T, N, 18), values=torch.zeros(T, N, 2),
                  actions_log_prob=torch.zeros(T, N, 2), rewards=torch.zeros(T, N, 2), dones=torch.zeros(T, N, 1, dtype=torch.uint8))
        t0 = time.perf_counter()
        obs = self.obs
        for t in range(T):
            self.step_count += 1
            a = PO.policy_act(self.P, obs, torch.randn(N, 18))
            st["observations"][t] = obs
            st["actions"][t], st["values"][t], st["actions_log_prob"][t] = a["actions"], a["values"], a["log_prob"]
            self._load(self.sim_fn(self.step_count), a["actions"])
            obs, rew, arew, rst, ex = self.env.post_physics_step(self.rand_fn(self.step_count), self.rt)
            st["rewards"][t] = PO.bootstrap_rewards(rew, arew, a["values"], self.env.s.time_out_buf, hp["gamma"])
            st["dones"][t] = rst.view(-1, 1).to(torch.uint8)
        self.obs = obs
        t1 = time.perf_counter()
        last = PO.critic_values(self.P, obs)
        st["returns"], st["advantages"] = PO.compute_returns(st["rewards"], st["values"], st["dones"], last, hp["gamma"], hp["lam"])
        t2 = time.perf_counter()
        idx = torch.randperm(N * T)
        logs = PO.ppo_update(self.P, self.opt, st, idx, hp, self.counter)
        self.counter += 1
        t3 = time.perf_counter()
        return dict(rollout=t1 - t0, gae=t2 - t1, update=t3 - t2, total=t3 - t0, logs=logs)
