"""Host-side mirror of the widowGo1 task's per-step surface, backed by the fused CUDA kernel.

`FusedWidowGo1Core` owns the task state that `WidowGo1._init_buffers` creates
(legged_gym/legged_gym/envs/widowGo1/widowGo1.py:498-672, cited WG:line) and exposes it under
the reference's attribute names (as views into two packed per-env rows, see include/dwbc.h),
so code written against the reference env (`OnPolicyRunner`, logging, play scripts) keeps
working.  `post_physics_step()` is ONE launch of `dwbc_post_physics_step`; `step()` keeps the
reference's 6-tuple (WG:1199).  The physics call itself stays outside (Isaac Gym); see
INTEGRATION.md for the subclass that plugs this into the real `WidowGo1`.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from .config import METRIC_NAMES, RAND_COLS, TERM_ID, CommandCurriculum, WidowGo1Params

CHECKPOINT_VERSION = 1          # layout of FusedWidowGo1Core.state_dict()
# the task state a checkpoint holds, by checkpoint name (load_state's where it has one) -> attribute; simulator-owned tensors (bind_sim)
# are the simulator's to save, and the per-env slots of ended episodes (_stats_scratch) are written before they are read
_CHECKPOINT = dict(actions="actions", action_history_buf="action_history_buf", goal_state="_goal_state", derived_state="_derived_state",
                   episode_length_buf="_episode_length", obs_history_buf="_hist", episode_sums="_sums", episode_stats="_stats",
                   mass_params="mass_params_tensor", friction="friction_coeffs_tensor", motor_strength="motor_strength",
                   env_origins="env_origins", box_env_origins_delta_y="box_env_origins_delta_y", terrain_levels="terrain_levels",
                   terrain_types="terrain_types", terrain_origins="terrain_origins", measured_heights="measured_heights",
                   heights_obs="heights_obs", rew_buf="rew_buf", arm_rew_buf="arm_rew_buf", reset_buf="reset_buf",
                   time_out_buf="time_out_buf")
_CURRICULUM_RANGES = ("lin_vel_x_ranges", "ang_vel_yaw_ranges", "goal_ee_l_ranges", "goal_ee_p_ranges", "goal_ee_y_ranges")


def make_env_cfg(p: WidowGo1Params, sums_stride: int) -> L.EnvCfg:
    c = L.EnvCfg()
    c.abi_version = L.ABI_VERSION
    c.num_envs, c.num_dofs, c.num_actions = p.num_envs, p.num_dofs, p.num_actions
    c.num_bodies_p1, c.gripper_idx = p.num_bodies + 1, p.gripper_idx
    c.num_prop, c.num_priv, c.history_len, c.num_obs = p.num_prop, p.num_priv, p.history_len, p.num_obs
    c.action_hist_len = p.action_hist_len
    for i in range(4):
        c.feet_idx[i] = p.feet_indices[i]
        c.feet_perm[i] = p.feet_perm()[i]
    if len(p.penalized_contact_indices) > L.MAX_IDX or len(p.termination_contact_indices) > L.MAX_IDX:
        raise L.DwbcError("too many contact bodies for the ABI struct")
    c.n_penalized = len(p.penalized_contact_indices)
    for i, v in enumerate(p.penalized_contact_indices):
        c.penalized_idx[i] = v
    c.n_term_contact = len(p.termination_contact_indices)
    for i, v in enumerate(p.termination_contact_indices):
        c.term_contact_idx[i] = v
    for i, v in enumerate(p.ig2raisim()):
        c.ig2raisim[i] = v
    c.waist_dof = p.num_dofs - 8                                        # WG:970
    c.goal_is_cart = int(p.command_mode == "cart")
    c.max_episode_length = int(p.max_episode_length)
    c.resample_interval = p.resample_interval
    if not 0 <= p.num_collision_check_samples <= len(c.collision_t):
        raise L.DwbcError(f"num_collision_check_samples = {p.num_collision_check_samples}: the kernels take 0 .. {len(c.collision_t)} "
                          f"collision samples per path")
    c.n_collision_samples, c.max_goal_tries = p.num_collision_check_samples, 10
    c.only_positive_rewards = int(p.only_positive_rewards)
    slots = p.sum_slots()
    for which, n_attr, t_attr, s_attr in (("leg", "n_leg_terms", "leg_term", "leg_slot"), ("arm", "n_arm_terms", "arm_term", "arm_slot")):
        terms = p.active_terms(which)
        if len(terms) > L.MAX_TERMS:
            raise L.DwbcError("too many active reward terms for the ABI struct")
        setattr(c, n_attr, len(terms))
        for i, t in enumerate(terms):
            if t not in TERM_ID:
                raise L.DwbcError(f"reward term '{t}' has no kernel implementation")
            getattr(c, t_attr)[i] = TERM_ID[t]
            getattr(c, s_attr)[i] = slots.index(t)
    c.termination_slot = slots.index("termination") if "termination" in slots else -1
    c.n_sum_slots, c.sums_stride = len(slots), sums_stride
    c.measure_heights = int(p.measure_heights)
    c.n_height_x, c.n_height_y = len(p.measured_points_x), len(p.measured_points_y)
    c.terrain_rows, c.terrain_cols = p.tot_rows, p.tot_cols
    c.terrain_curriculum, c.max_terrain_level, c.terrain_n_types = int(p.terrain_curriculum), p.max_terrain_level, p.terrain_num_cols
    for i in range(p.num_dofs):
        c.default_dof_pos[i] = p.default_dof_pos[i]
        c.dof_pos_lower[i], c.dof_pos_upper[i] = p.dof_pos_limits[i]
        c.dof_vel_limits[i], c.torque_limits[i] = p.dof_vel_limits[i], p.torque_limits[i]
    c.obs_scale_lin_vel, c.obs_scale_ang_vel = p.obs_scale_lin_vel, p.obs_scale_ang_vel
    c.obs_scale_dof_pos, c.obs_scale_dof_vel, c.obs_scale_height = p.obs_scale_dof_pos, p.obs_scale_dof_vel, p.obs_scale_height
    c.clip_obs = p.clip_observations
    c.term_roll, c.term_pitch, c.term_z = p.term_roll, p.term_pitch, p.term_z
    c.lin_vel_x_clip, c.ang_vel_yaw_clip = p.lin_vel_x_clip, p.ang_vel_yaw_clip
    tt = torch.linspace(0, 1, p.num_collision_check_samples)           # WG:586, exact torch values
    for i in range(3):
        c.collision_lower[i], c.collision_upper[i] = p.collision_lower_limits[i], p.collision_upper_limits[i]
        c.sphere_error_scale[i], c.orn_error_scale[i] = p.sphere_error_scale[i], p.orn_error_scale[i]
        c.delta_orn_lo[i] = p.final_delta_orn[i][0]
        c.delta_orn_span[i] = p.final_delta_orn[i][1] - p.final_delta_orn[i][0]
    for i in range(p.num_collision_check_samples):
        c.collision_t[i] = float(tt[i])
    c.underground_limit, c.z_invariant_offset = p.underground_limit, p.z_invariant_offset
    c.tracking_sigma, c.tracking_ee_sigma = p.tracking_sigma, p.tracking_ee_sigma
    c.base_height_target, c.max_contact_force = p.base_height_target, p.max_contact_force
    c.soft_dof_vel_limit, c.soft_torque_limit, c.dt, c.max_episode_length_s = p.soft_dof_vel_limit, p.soft_torque_limit, p.dt, p.max_episode_length_s
    for i in range(13):
        c.base_init_state[i] = p.base_init_state[i]
    c.origin_perturb[0], c.origin_perturb[1] = -p.origin_perturb_range, p.origin_perturb_range - (-p.origin_perturb_range)
    c.init_vel_perturb[0], c.init_vel_perturb[1] = -p.init_vel_perturb_range, p.init_vel_perturb_range - (-p.init_vel_perturb_range)
    c.box_x, c.box_z = p.box_env_origins_x, p.box_env_origins_z
    c.push_vel[0], c.push_vel[1] = -p.max_push_vel_xy, p.max_push_vel_xy - (-p.max_push_vel_xy)
    c.dof_reset[0], c.dof_reset[1] = 0.8, 1.2 - 0.8
    for i, v in enumerate(p.measured_points_x):
        c.height_x[i] = v
    for i, v in enumerate(p.measured_points_y):
        c.height_y[i] = v
    c.border_size, c.horizontal_scale, c.vertical_scale = p.border_size, p.horizontal_scale, p.vertical_scale
    c.terrain_env_length = p.terrain_env_length
    return c


class FusedWidowGo1Core:
    """Task state + fused post-physics step for one env shard on one GPU."""

    def __init__(self, p: WidowGo1Params, device="cuda:0", state: Optional[Dict[str, np.ndarray]] = None, seed: int = 0,
                 sync_stats: bool = True, generic_kernel: bool = False):
        self.p, self.cfg_params = p, p
        self.device = torch.device(device)
        self.num_envs, self.num_obs, self.num_actions = p.num_envs, p.num_obs, p.num_actions
        self.num_privileged_obs = None
        self.max_episode_length = p.max_episode_length
        self.dt = p.dt
        self.seed, self.sync_stats = seed, sync_stats
        self.common_step_counter = 0
        self._lib = L.lib()
        N, dev = p.num_envs, self.device
        z = lambda *s, dtype=torch.float: torch.zeros(*s, dtype=dtype, device=dev)  # noqa: E731
        # --- Isaac-Gym-owned tensors (caller may re-bind them to gymtorch views with `bind_sim`) ---
        self._root_states = z(N, 2, 13)
        self.dof_state = z(N * p.num_dofs, 2)
        self._rigid_body_state = z(N, p.num_bodies + 1, 13)
        self._contact_forces = z(N, p.num_bodies + 1, 3)
        self.force_sensor_tensor = z(N, 4, 6)
        self.torques = z(N, p.num_dofs)
        self.actions = z(N, p.num_actions)
        self.action_history_buf = z(N, p.action_hist_len, p.num_actions)
        # --- per-env constants ---
        self.mass_params_tensor, self.friction_coeffs_tensor = z(N, 5), z(N, 1)
        self.motor_strength = torch.ones(N, p.num_actions, device=dev)
        self.env_origins, self.box_env_origins_delta_y = z(N, 3), z(N)
        # --- packed task state ---
        self._goal_state, self._derived_state = z(N, L.GS), z(N, L.DS)
        self._episode_length = z(N, dtype=torch.long)
        self._hist = z(N, p.history_len, p.num_prop)
        self.sum_names = p.sum_slots()
        self._nslots = len(self.sum_names) + len(METRIC_NAMES)
        self._sums_stride = (self._nslots + 3) // 4 * 4
        self._sums = z(N, self._sums_stride)
        self.episode_sums = {k: self._sums[:, i] for i, k in enumerate(self.sum_names)}
        self.episode_metric_sums = {k: self._sums[:, len(self.sum_names) + i] for i, k in enumerate(METRIC_NAMES)}
        self._stats = z(1 + self._sums_stride)
        self._stats_scratch = z(N, self._sums_stride)    # per-env slots of the ended episodes' sums (episode_scratch)
        self._pd = None
        # --- terrain ---
        self.height_samples = None
        npts = p.num_height_points
        self.measured_heights = z(N, npts) if p.measure_heights else None
        self.heights_obs = z(N, npts) if p.measure_heights else None
        self.terrain_levels, self.terrain_types = z(N, dtype=torch.long), z(N, dtype=torch.long)
        self.terrain_origins = z(p.max_terrain_level, p.terrain_num_cols, 3)
        # --- outputs ---
        self._obs_own = z(N, p.num_obs)
        self.obs_buf = self._obs_own
        self.privileged_obs_buf = None
        self.rew_buf, self.arm_rew_buf = z(N), z(N)
        self.reset_buf = torch.ones(N, dtype=torch.bool, device=dev)
        self.time_out_buf = z(N, dtype=torch.bool)
        self._rand = None
        self.extras = {"episode": {}}
        self._raisim2ig = torch.tensor(p.raisim2ig(p.num_actions), dtype=torch.int32, device=dev)
        self.curriculum = CommandCurriculum(p)
        self._cfg = make_env_cfg(p, self._sums_stride)
        self._buf = L.EnvBuffers()
        self._args = L.StepArgs()
        self._dev_step = None          # device DwbcStepDevice of a captured rollout (set_device_step)
        # True: always the warp-per-env kernel, which also runs by itself when N is not a multiple of 32 or a state row block is not
        # 16-byte aligned (the observation target and the history must be 16-byte aligned for both kernels)
        self._args.generic_kernel = int(generic_kernel)
        self._leg_terms, self._arm_terms = p.active_terms("leg"), p.active_terms("arm")
        if state is not None:
            self.load_state(state)
        self._bind()
        self._refresh_args()

    # ------------------------------------------------------------------ reference-named views
    def _gs(self, name, n=1):
        c = L.GS_COL[name]
        return self._goal_state[:, c] if n == 1 else self._goal_state[:, c:c + n]

    def _ds(self, name, n):
        c = L.DS_COL[name]
        return self._derived_state[:, c:c + n]

    commands = property(lambda s: s._gs("commands", 3))
    goal_timer = property(lambda s: s._gs("goal_timer"))
    traj_timesteps = property(lambda s: s._gs("traj_timesteps"))
    traj_total_timesteps = property(lambda s: s._gs("traj_total_timesteps"))
    ee_start_sphere = property(lambda s: s._gs("ee_start_sphere", 3))
    ee_goal_sphere = property(lambda s: s._gs("ee_goal_sphere", 3))
    ee_goal_cart = property(lambda s: s._gs("ee_goal_cart", 3))
    curr_ee_goal_sphere = property(lambda s: s._gs("curr_ee_goal_sphere", 3))
    curr_ee_goal_cart = property(lambda s: s._gs("curr_ee_goal_cart", 3))
    ee_goal_delta_orn_euler = property(lambda s: s._gs("ee_goal_delta_orn_euler", 3))
    ee_goal_orn_euler = property(lambda s: s._gs("ee_goal_orn_euler", 3))
    curr_ee_goal = property(lambda s: s.curr_ee_goal_cart if s.p.command_mode == "cart" else s.curr_ee_goal_sphere)
    base_lin_vel = property(lambda s: s._ds("base_lin_vel", 3))
    base_ang_vel = property(lambda s: s._ds("base_ang_vel", 3))
    base_yaw_euler = property(lambda s: s._ds("base_yaw_euler", 3))
    base_yaw_quat = property(lambda s: s._ds("base_yaw_quat", 4))
    last_root_vel = property(lambda s: s._ds("last_root_vel", 6))
    feet_air_time = property(lambda s: s._ds("feet_air_time", 4))
    last_contacts = property(lambda s: s._ds("last_contacts", 4))
    last_actions = property(lambda s: s._ds("last_actions", s.p.num_actions))
    last_dof_vel = property(lambda s: s._ds("last_dof_vel", s.p.num_dofs))
    root_states = property(lambda s: s._root_states[:, 0, :])
    box_root_state = property(lambda s: s._root_states[:, 1, :])
    base_quat = property(lambda s: s._root_states[:, 0, 3:7])
    dof_pos = property(lambda s: s.dof_state.view(s.num_envs, s.p.num_dofs, 2)[..., 0])
    dof_vel = property(lambda s: s.dof_state.view(s.num_envs, s.p.num_dofs, 2)[..., 1])
    rigid_body_state = property(lambda s: s._rigid_body_state[:, :-1, :])
    contact_forces = property(lambda s: s._contact_forces[:, :-1, :])
    ee_pos = property(lambda s: s._rigid_body_state[:, s.p.gripper_idx, :3])

    @property
    def obs_history_buf(self):
        """[N, history_len, num_prop] proprioception history, stored unclipped as in the reference.  The TMA kernel keeps a per-env
        count of the most recent history rows known to lie within +-clip_observations (derived_state column 27) and skips the
        clipping of obs[:, 100:] while that count covers the whole history; `load_state` resets the count.  A write into this
        tensor from outside (anything but `load_state`) must not store a value beyond +-clip_observations, or the next
        observations may carry it unclipped."""
        return self._hist

    @property
    def episode_length_buf(self):
        return self._episode_length

    @episode_length_buf.setter
    def episode_length_buf(self, v):        # the runner re-binds this attribute (OPR:107-108)
        self._episode_length.copy_(v.to(self._episode_length.dtype))

    # ------------------------------------------------------------------ state loading / binding
    def load_state(self, st: Dict[str, np.ndarray]):
        """Load reference-named arrays (numpy or torch) such as synth.initial_env_state()."""
        T = lambda a: torch.as_tensor(np.ascontiguousarray(a) if isinstance(a, np.ndarray) else a).to(self.device)  # noqa: E731
        direct = dict(root_states="_root_states", dof_state="dof_state", rigid_body_state="_rigid_body_state",
                      contact_forces="_contact_forces", force_sensor="force_sensor_tensor", torques="torques",
                      action_history_buf="action_history_buf", mass_params="mass_params_tensor",
                      friction="friction_coeffs_tensor", motor_strength="motor_strength", env_origins="env_origins",
                      box_env_origins_delta_y="box_env_origins_delta_y", obs_history_buf="_hist",
                      episode_length_buf="_episode_length", terrain_levels="terrain_levels", terrain_types="terrain_types",
                      terrain_origins="terrain_origins", actions="actions")
        for k, v in st.items():
            if k in direct:
                getattr(self, direct[k]).copy_(T(v).reshape(getattr(self, direct[k]).shape))
            elif k in L.GS_COL:
                t = T(v).float()
                self._gs(k, 1 if t.dim() == 1 else t.shape[1]).copy_(t)
            elif k in L.DS_COL:
                t = T(v).float()
                self._ds(k, t.shape[1]).copy_(t)
            elif k == "height_samples":
                self.height_samples = T(v).to(torch.int16).contiguous()
        if "obs_history_buf" in st:
            self._derived_state[:, 27] = 0.0          # DWBC_DS_OOB_AGE: unknown history -> kernel takes the clipping path for H steps
        if "actions" not in st and "action_history_buf" in st:
            self.actions.copy_(self.action_history_buf[:, 1])      # [:, -action_delay-1] with AH = delay+2 (WG:541,1167)
        if getattr(self, "_bound", False):
            self._bind()                                           # height_samples is a NEW tensor: refresh the kernel's pointer table

    def bind_sim(self, **tensors):
        """Re-bind Isaac-Gym-owned buffers to external tensors (zero-copy gymtorch views):
        root_states [N,2,13], dof_state, rigid_body_state, contact_forces, force_sensor, torques."""
        names = dict(root_states="_root_states", dof_state="dof_state", rigid_body_state="_rigid_body_state",
                     contact_forces="_contact_forces", force_sensor="force_sensor_tensor", torques="torques")
        for k, t in tensors.items():
            setattr(self, names[k], t)
        self._bind()

    def set_obs_target(self, tensor: Optional[torch.Tensor]):
        """Direct the kernel's observation output to `tensor` ([N, >=num_obs] row-major), e.g. a row
        of RolloutStorage.observations (SURVEY f2: saves the RS:98 copy).  The kernels write whole rows in 16-byte vectors, so the
        target must be float32 on this core's device with unit column stride, a 16-byte-aligned start and a row stride that is a
        multiple of 4 floats; anything else raises DwbcError here instead of reaching the kernel."""
        if tensor is not None:
            if tensor.dtype != torch.float32 or tensor.device.type != self.device.type or \
                    (self.device.index is not None and tensor.device.index != self.device.index):
                raise L.DwbcError(f"obs target must be float32 on {self.device}, got {tensor.dtype} on {tensor.device}")
            if tensor.dim() != 2 or tensor.shape[0] != self.num_envs or tensor.shape[1] < self.num_obs or tensor.stride(1) != 1:
                raise L.DwbcError(f"obs target must be [{self.num_envs}, >={self.num_obs}] with unit column stride, "
                                  f"got shape {tuple(tensor.shape)} strides {tensor.stride()}")
            if tensor.data_ptr() % 16 or tensor.stride(0) % 4:
                raise L.DwbcError(f"obs target must start 16-byte aligned with a row stride that is a multiple of 4 floats, "
                                  f"got address {tensor.data_ptr():#x} and row stride {tensor.stride(0)}")
        self.obs_buf = self._obs_own if tensor is None else tensor
        self._buf.obs_buf = self.obs_buf.data_ptr()
        self._buf.obs_stride = self.obs_buf.stride(0)

    def set_transition_target(self, values: Optional[torch.Tensor], rewards: Optional[torch.Tensor] = None, dones: Optional[torch.Tensor] = None,
                              gamma: float = 0.0):
        """Direct-to-storage transition (SURVEY f2): with `rewards` = row t of RolloutStorage.rewards [N,2] (and `values` = the values
        PPO.act wrote for this step, `dones` = row t of RolloutStorage.dones, uint8) the post-physics kernel itself performs
        PPO.process_env_step's reward path (PPO:130-134) and the dones store (RS:102); FusedPPO.process_env_step recognises the rows and
        launches nothing.  `set_transition_target(None)` switches it off."""
        b = self._buf
        if values is None or rewards is None:
            b.store_values = b.store_rewards = b.store_dones = None
            self._stored_rows = None
            return
        b.store_values, b.store_rewards = L.ptr(values, torch.float32), L.ptr(rewards, torch.float32)
        b.store_dones = None if dones is None else L.ptr(dones, torch.uint8)
        b.store_gamma = float(gamma)
        self._stored_rows = (rewards.data_ptr(), None if dones is None else dones.data_ptr())

    def _bind(self):
        self._bound = True
        b, P = self._buf, L.ptr
        b.root_states, b.dof_state = P(self._root_states), P(self.dof_state)
        b.rigid_body_state, b.contact_forces = P(self._rigid_body_state), P(self._contact_forces)
        b.force_sensor, b.torques, b.actions = P(self.force_sensor_tensor), P(self.torques), P(self.actions)
        b.action_history = P(self.action_history_buf)
        b.mass_params, b.friction, b.motor_strength = P(self.mass_params_tensor), P(self.friction_coeffs_tensor), P(self.motor_strength)
        b.env_origins, b.box_env_origins_delta_y = P(self.env_origins), P(self.box_env_origins_delta_y)
        b.goal_state, b.derived_state, b.episode_length = P(self._goal_state), P(self._derived_state), P(self._episode_length)
        b.obs_history, b.episode_sums = P(self._hist), P(self._sums)
        b.height_samples, b.measured_heights, b.heights_obs = P(self.height_samples), P(self.measured_heights), P(self.heights_obs)
        b.terrain_levels, b.terrain_types, b.terrain_origins = P(self.terrain_levels), P(self.terrain_types), P(self.terrain_origins)
        b.obs_buf, b.obs_stride = self.obs_buf.data_ptr(), self.obs_buf.stride(0)
        b.rew_buf, b.arm_rew_buf = P(self.rew_buf), P(self.arm_rew_buf)
        b.reset_buf, b.time_out_buf, b.episode_stats = P(self.reset_buf), P(self.time_out_buf), P(self._stats)
        b.episode_scratch = P(self._stats_scratch)

    # ------------------------------------------------------------------ checkpoint of the task state
    def _checkpoint_tensors(self) -> Dict[str, torch.Tensor]:
        t = {k: getattr(self, a) for k, a in _CHECKPOINT.items() if getattr(self, a) is not None}
        t["obs_buf"] = self.obs_buf[:, :self.num_obs]                   # the current observation, wherever it is targeted
        return t

    def state_dict(self) -> dict:
        """Everything this core owns that the post-physics step reads or advances: the packed goal / derived rows (all columns,
        the TMA kernel's out-of-range history counter included), history, action FIFO, episode lengths, sums and unread statistics,
        per-env constants, terrain state (and the height field when heights are measured), the current observation and the last
        step's outputs, `common_step_counter`, `seed` and the command curriculum.  The simulator's tensors are not included."""
        cur = self.curriculum
        t = {k: v.clone() for k, v in self._checkpoint_tensors().items()}
        if self.p.measure_heights and self.height_samples is not None:
            t["height_samples"] = self.height_samples.clone()
        return dict(version=CHECKPOINT_VERSION, cfg=torch.frombuffer(bytearray(bytes(self._cfg)), dtype=torch.uint8), tensors=t,
                    common_step_counter=self.common_step_counter, seed=self.seed,
                    curriculum=dict(update_counter=cur.update_counter, **{k: [float(x) for x in getattr(cur, k)] for k in _CURRICULUM_RANGES},
                                    reward_scales={k: float(v) for k, v in cur.reward_scales.items()},
                                    arm_reward_scales={k: float(v) for k, v in cur.arm_reward_scales.items()}))

    def load_state_dict(self, sd: dict):
        """Restore a state_dict() in place.  A checkpoint of a core built with another DwbcEnvCfg (envs, history length, reward
        terms, sums layout, ...) or of another format version raises DwbcError before anything is copied.  No tensor is re-bound,
        except a height field on a core that has none yet: it is allocated and bound as `load_state` does (a captured rollout then
        re-captures)."""
        keys = {"version", "cfg", "tensors", "common_step_counter", "seed", "curriculum"}
        if not isinstance(sd, dict) or sd.get("version") != CHECKPOINT_VERSION or set(sd) != keys:
            raise L.DwbcError(f"not a FusedWidowGo1Core checkpoint of format version {CHECKPOINT_VERSION}: "
                              f"version {sd.get('version') if isinstance(sd, dict) else None}")
        if bytes(sd["cfg"].cpu().numpy()) != bytes(self._cfg):
            raise L.DwbcError("the checkpoint was taken on a core built with another DwbcEnvCfg (envs, history, reward terms, sums layout, ...)")
        src, own = sd["tensors"], self._checkpoint_tensors()
        hs = src.get("height_samples")
        if set(src) - {"height_samples"} != set(own) or (hs is not None and not self.p.measure_heights):
            raise L.DwbcError(f"the checkpoint holds the tensors {sorted(src)}, this core {sorted(own)}")
        for k, dst in own.items():
            if src[k].shape != dst.shape or src[k].dtype != dst.dtype:
                raise L.DwbcError(f"{k}: {src[k].dtype}{list(src[k].shape)} in the checkpoint, {dst.dtype}{list(dst.shape)} in this core")
        if hs is not None and (hs.dtype != torch.int16 or tuple(hs.shape) != (self.p.tot_rows, self.p.tot_cols)):
            raise L.DwbcError(f"height_samples: {hs.dtype}{list(hs.shape)}, not int16[{self.p.tot_rows}, {self.p.tot_cols}]")
        cur, c = self.curriculum, sd["curriculum"]
        if set(c["reward_scales"]) != set(cur.reward_scales) or set(c["arm_reward_scales"]) != set(cur.arm_reward_scales):
            raise L.DwbcError("the checkpoint's curriculum scales other reward terms")
        for k, dst in own.items():
            dst.copy_(src[k])
        if hs is not None:
            if self.height_samples is None or self.height_samples.shape != hs.shape:
                self.height_samples = hs.to(self.device, copy=True).contiguous()
                self._bind()
            else:
                self.height_samples.copy_(hs)
        self.common_step_counter, self.seed = int(sd["common_step_counter"]), int(sd["seed"])
        cur.update_counter = int(c["update_counter"])
        for k in _CURRICULUM_RANGES:
            setattr(cur, k, np.array(c[k], dtype=np.float64))
        cur.reward_scales, cur.arm_reward_scales = dict(c["reward_scales"]), dict(c["arm_reward_scales"])
        self._refresh_args()

    # ------------------------------------------------------------------ curriculum (WG:678-692)
    def update_command_curriculum(self):
        self.curriculum.update()
        self._refresh_args()

    def _refresh_args(self):
        a, cur = self._args, self.curriculum

        def pair(dst, rng):
            dst[0], dst[1] = float(rng[0]), float(rng[1] - rng[0])       # span formed in float64 like the reference
        pair(a.lin_vel_x, cur.lin_vel_x_ranges)
        pair(a.ang_vel_yaw, cur.ang_vel_yaw_ranges)
        pair(a.goal_l, cur.goal_ee_l_ranges)
        pair(a.goal_p, cur.goal_ee_p_ranges)
        pair(a.goal_y, cur.goal_ee_y_ranges)
        for i, t in enumerate(self._leg_terms):
            a.leg_scale[i] = cur.reward_scales[t]
        for i, t in enumerate(self._arm_terms):
            a.arm_scale[i] = cur.arm_reward_scales[t]
        a.leg_termination_scale = cur.reward_scales.get("termination", 0.0)
        a.arm_termination_scale = cur.arm_reward_scales.get("termination", 0.0)

    # ------------------------------------------------------------------ step
    def pre_physics_step(self, policy_actions: torch.Tensor) -> torch.Tensor:
        """WG:1162-1173: permute raisim->IG, clip, FIFO push, delayed action -> self.actions."""
        p = self.p
        if p.action_delay < 0 or p.action_hist_len != p.action_delay + 2:
            raise L.DwbcError("action_delay = -1 (no delay FIFO, WG:1166) / a history length other than action_delay + 2 is not implemented")
        delay_row = p.action_hist_len - p.action_delay - 1              # action_history_buf[:, -action_delay - 1] after the shift (WG:1167-1168)
        L.check(self._lib.dwbc_pre_physics_actions(L.ptr(policy_actions.contiguous(), torch.float32), L.ptr(self._raisim2ig), float(p.clip_actions),
                                                   L.ptr(self.action_history_buf), L.ptr(self.actions), p.num_envs, p.num_actions,
                                                   p.action_hist_len, delay_row, L.stream_ptr()), "dwbc_pre_physics_actions")
        return self.actions

    def compute_torques(self, actions: Optional[torch.Tensor] = None) -> torch.Tensor:
        """WG:1262-1295 `_compute_torques` (PD controller; the reference calls it `decimation` times per policy step, WG:1175-1183,
        with the dof state refreshed in between).  Writes `self.torques` [N, n_dof] and returns it."""
        p = self.p
        if self._pd is None:
            pd = L.PdCfg()
            pd.n_dof, pd.n_act, pd.wrap_dof = p.num_dofs, p.num_actions, p.num_actions - 8     # column -8 of the 18-wide tensor (WG:1279)
            for k, src in (("p_gains", p.p_gains), ("d_gains", p.d_gains), ("action_scale", p.action_scale),
                           ("default_dof_pos", p.default_dof_pos), ("torque_limits", p.torque_limits)):
                arr = getattr(pd, k)
                for i, v in enumerate(src):
                    arr[i] = float(v)
            self._pd = pd
        a = self.actions if actions is None else actions.contiguous()
        L.check(self._lib.dwbc_compute_torques(C.addressof(self._pd), L.ptr(a), L.ptr(self.dof_state), L.ptr(self.motor_strength),
                                               L.ptr(self.torques), p.num_envs, L.stream_ptr()), "dwbc_compute_torques")
        return self.torques

    def post_physics_step(self, rand: Optional[torch.Tensor] = None):
        """WG:865-915 after the gym.refresh_* calls.  `rand` ([N, RAND_COLS] uniforms) selects table
        mode; otherwise the kernel draws Philox uniforms keyed by (seed, common_step_counter)."""
        self.common_step_counter += 1
        a = self._args
        a.rand_uniform = None if rand is None else L.ptr(rand)
        a.seed, a.step = self.seed, self.common_step_counter
        a.do_push = int(self.p.push_robots and (self.common_step_counter % self.p.push_interval == 0))
        self._pushed = bool(a.do_push)
        self.reset_count = None
        if self.sync_stats:
            self._stats.zero_()        # per-step episode statistics (WG:743-750); without them the accumulators are read by episode_stats()
        if self._dev_step is None:
            L.check(self._lib.dwbc_post_physics_step(C.addressof(self._cfg), C.addressof(self._buf), C.addressof(a), L.stream_ptr()),
                    "dwbc_post_physics_step")
        else:
            L.check(self._lib.dwbc_post_physics_step_device(C.addressof(self._cfg), C.addressof(self._buf), C.addressof(a),
                                                            L.ptr(self._dev_step, torch.uint8), L.stream_ptr()), "dwbc_post_physics_step_device")
        self.extras["time_outs"] = self.time_out_buf
        self.extras["dwbc_stored_rows"] = getattr(self, "_stored_rows", None)
        if self.sync_stats:
            self._fill_episode_extras()

    def step_record(self) -> torch.Tensor:
        """The DwbcStepDevice of the next post_physics_step (uint8 host tensor): the step, the push interval and the curriculum values
        this core would pass by value.  Copied to the device record given to `set_device_step`, it lets a captured post_physics_step
        read them at run time; each call then advances the step on the device."""
        r, a = L.StepDevice(), self._args
        r.step = self.common_step_counter + 1
        r.push_interval = int(self.p.push_interval) if self.p.push_robots else 0
        first, end = L.StepArgs.lin_vel_x.offset, L.StepArgs.generic_kernel.offset
        C.memmove(C.addressof(r) + L.StepDevice.lin_vel_x.offset, C.addressof(a) + first, end - first)
        return torch.frombuffer(bytearray(bytes(r)), dtype=torch.uint8)

    def set_device_step(self, record: Optional[torch.Tensor]):
        """Make post_physics_step launch through dwbc_post_physics_step_device with this device DwbcStepDevice ([sizeof] uint8 CUDA
        tensor) or, with None, through dwbc_post_physics_step with the host fields again."""
        if record is not None and (record.dtype != torch.uint8 or record.numel() != C.sizeof(L.StepDevice)):
            raise L.DwbcError(f"the device step record is a uint8 tensor of {C.sizeof(L.StepDevice)} bytes")
        self._dev_step = record

    def episode_stats(self, reset: bool = True):
        """`extras['episode']` over every episode that ended since the last call (one D2H read; for sync_stats=False loops that log once per
        iteration instead of syncing on every step like WG:705)."""
        self._fill_episode_extras()
        if reset:
            self._stats.zero_()
        return self.extras["episode"]

    def _fill_episode_extras(self, st=None, coeffs=None):
        """extras['episode'] (WG:743-750) from the stats block `st` on the host (default: one D2H read of the device block; the reference
        syncs on len(env_ids) at WG:705 as well) and the curriculum coefficients `coeffs` (default: the current ones)."""
        st = self._stats.cpu() if st is None else st
        cnt = float(st[0])
        if cnt > 0:
            ep = {}
            for i, k in enumerate(self.sum_names):
                ep["rew_" + k] = st[1 + i] / cnt / self.p.max_episode_length_s
            for i, k in enumerate(METRIC_NAMES):
                ep["metric_" + k] = st[1 + len(self.sum_names) + i] / cnt / self.p.max_episode_length_s
            self.extras["episode"] = ep
        self.extras["episode"].update(self._curriculum_coeffs() if coeffs is None else coeffs)
        self.reset_count = int(cnt)

    def _curriculum_coeffs(self):
        """The command-curriculum values _fill_episode_extras adds to extras['episode']."""
        cur = self.curriculum
        return dict(coeff_lin_vel_x_upper_bound=cur.lin_vel_x_ranges[1], coeff_lin_vel_x_lower_bound=cur.lin_vel_x_ranges[0],
                    coeff_ang_vel_yaw_upper_bound=cur.ang_vel_yaw_ranges[1], coeff_ang_vel_yaw_lower_bound=cur.ang_vel_yaw_ranges[0],
                    coeff_tracking_ang_vel_yaw_exp=cur.reward_scales.get("tracking_ang_vel_yaw_exp", 0.0))

    @property
    def sim_state_dirty(self) -> bool:
        """True when the last post_physics_step changed simulator-owned state (`_root_states` on push steps, WG:804-814; `_root_states`
        and `dof_state` of reset envs, WG:757-828), i.e. when the caller owes Isaac Gym the `gym.set_*_tensor` calls the reference
        issues at WG:787,813,827.  Without per-step statistics (`sync_stats=False`: no host read of the reset count) every step counts
        as dirty -- writing back an unchanged tensor is harmless, skipping a changed one silently drops the push / reset."""
        if getattr(self, "_pushed", False) or not self.sync_stats:
            return True
        return bool(self.reset_count)

    def step(self, actions: torch.Tensor, physics=None):
        """VecEnv.step (WG:1156-1199).  `physics(env)` stands for the decimated Isaac Gym loop
        (WG:1177-1192): it must leave fresh sim tensors + torques in the bound buffers."""
        self.pre_physics_step(actions)
        if physics is not None:
            physics(self)
        self.post_physics_step()
        return self.obs_buf, self.privileged_obs_buf, self.rew_buf, self.arm_rew_buf, self.reset_buf, self.extras

    def get_observations(self):
        return self.obs_buf

    def get_privileged_observations(self):
        return self.privileged_obs_buf

    def fill_uniform(self, step: int) -> torch.Tensor:
        """The uniform table the in-kernel Philox stream produces for `step` (for parity checks)."""
        out = torch.empty(self.num_envs, RAND_COLS, device=self.device)
        L.check(self._lib.dwbc_fill_uniform(L.ptr(out), self.num_envs, self.seed, step, L.stream_ptr()), "dwbc_fill_uniform")
        return out
