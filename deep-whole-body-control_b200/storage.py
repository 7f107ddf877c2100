"""Device-resident rollout storage with the reference's field names and shapes
(`RolloutStorage`, rsl_rl/rsl_rl/storage/rollout_storage.py:56-205, cited RS:line).

Differences that are invisible through the reference's surface:
* `observations` is a view of a [T+1, N, n_obs] buffer: the env kernel writes obs_{t+1} straight
  into row t+1 (no `RS:98` copy) and row T holds the bootstrap observation of `compute_returns`;
* `compute_returns` is one cooperative kernel (GAE scan + joint advantage normalisation);
* `mini_batch_generator` yields *index tensors*: rows are gathered inside the GEMM operand loads,
  never materialised.  The permutation is drawn once per update and reused for every epoch
  exactly like RS:163.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L
from . import shard


class FusedRolloutStorage:
    class Transition:
        def __init__(self):
            self.observations = self.critic_observations = self.actions = self.rewards = self.dones = None
            self.values = self.actions_log_prob = self.action_mean = self.action_sigma = self.hidden_states = None

        def clear(self):
            self.__init__()

    def __init__(self, num_envs, num_transitions_per_env, obs_shape, privileged_obs_shape, actions_shape, device="cuda:0"):
        if privileged_obs_shape[0] is not None:
            raise L.DwbcError("separate privileged observations are not used by widowGo1 (WGC:127: None)")
        self.device = torch.device(device)
        T, N = num_transitions_per_env, num_envs
        self.num_transitions_per_env, self.num_envs = T, N
        self.obs_shape, self.privileged_obs_shape, self.actions_shape = obs_shape, privileged_obs_shape, actions_shape
        z = lambda *s, dtype=torch.float: torch.zeros(*s, dtype=dtype, device=self.device)  # noqa: E731
        self._obs_all = z(T + 1, N, *obs_shape)
        self.observations = self._obs_all[:T]
        self.privileged_observations = None
        self.rewards, self.actions = z(T, N, 2), z(T, N, *actions_shape)
        self.dones = z(T, N, 1, dtype=torch.uint8)                       # RS:72
        self.actions_log_prob, self.values = z(T, N, 2), z(T, N, 2)
        self.returns, self.advantages = z(T, N, 2), z(T, N, 2)
        self.mu, self.sigma = z(T, N, *actions_shape), z(T, N, *actions_shape)
        self._stats = torch.zeros(L.GAE_STATS, dtype=torch.float64, device=self.device)   # (n, sum, sum sq), then dwbc_gae's partials
        self.step = 0
        self._lib = L.lib()
        self._c = L.Storage()
        self._c.observations, self._c.obs_stride = self.observations.data_ptr(), obs_shape[0]
        self._c.actions, self._c.values, self._c.returns = self.actions.data_ptr(), self.values.data_ptr(), self.returns.data_ptr()
        self._c.advantages, self._c.log_prob = self.advantages.data_ptr(), self.actions_log_prob.data_ptr()
        self._c.hist_latent, self._c.hist_latent_ld = None, 0
        self._hist_latent = None
        # RS:82-84: the reference always allocates the three torque-supervision tensors; here they exist (and the kernels' branch is on)
        # only after enable_torque_supervision()
        self.target_arm_torques = self.current_arm_dof_pos = self.current_arm_dof_vel = None

    def enable_torque_supervision(self, n_arm=6):
        """RS:82-84 / RS:108-111: [T, N, n_arm] targets of the arm torque-supervision loss (PPO:224-239)."""
        T, N = self.num_transitions_per_env, self.num_envs
        self.target_arm_torques, self.current_arm_dof_pos, self.current_arm_dof_vel = (
            torch.zeros(T, N, n_arm, device=self.device) for _ in range(3))
        self._c.target_arm_torques, self._c.current_arm_dof_pos = self.target_arm_torques.data_ptr(), self.current_arm_dof_pos.data_ptr()
        self._c.current_arm_dof_vel = self.current_arm_dof_vel.data_ptr()

    def set_hist_latent(self, z):
        """Precomputed history latent of every storage row [T*N, ld] (or None): see DwbcStorage.hist_latent."""
        self._hist_latent = z
        self._c.hist_latent, self._c.hist_latent_ld = (None, 0) if z is None else (z.data_ptr(), z.stride(0))

    def obs_row(self, t):
        return self._obs_all[t]

    def clear(self):
        self.step = 0

    def compute_returns(self, last_values, gamma, lam, world_size: int = 1, group=None):
        """RS:136-150.  With world_size > 1 the advantage statistics (n, sum, sum of squares) are
        all-reduced so the normalisation equals that of the union batch (SURVEY 8e)."""
        T, N = self.num_transitions_per_env, self.num_envs
        self._stats.zero_()
        fused = world_size == 1
        L.check(self._lib.dwbc_gae(L.ptr(self.rewards), L.ptr(self.values), L.ptr(self.dones), L.ptr(last_values.contiguous()),
                                   L.ptr(self.returns), L.ptr(self.advantages), L.ptr(self._stats), T, N, gamma, lam, int(fused),
                                   L.stream_ptr()), "dwbc_gae")
        if not fused:
            shard.allreduce_adv_stats_(self._stats[:3], world_size, group)
            L.check(self._lib.dwbc_normalize_advantages(L.ptr(self.advantages), L.ptr(self._stats), T * N * 2, L.stream_ptr()),
                    "dwbc_normalize_advantages")

    def draw_indices(self, num_mini_batches, generator=None):
        batch = self.num_envs * self.num_transitions_per_env
        mbs = batch // num_mini_batches
        return torch.randperm(num_mini_batches * mbs, device=self.device, generator=generator), mbs   # RS:161-163

    def mini_batch_generator(self, num_mini_batches, num_epochs=8, indices=None):
        """Yields (batch_idx int64 [M]) per (epoch, mini-batch) in the order of RS:182-188."""
        if indices is None:
            indices, mbs = self.draw_indices(num_mini_batches)
        else:
            mbs = indices.numel() // num_mini_batches
        for _ in range(num_epochs):
            for i in range(num_mini_batches):
                yield indices[i * mbs:(i + 1) * mbs]

    def c_struct_ptr(self):
        return C.addressof(self._c)
