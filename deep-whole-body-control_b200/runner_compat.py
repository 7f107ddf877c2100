"""Drop-in classes for the reference's own driver code: what `OnPolicyRunner.__init__` / `learn` (rsl_rl/runners/on_policy_runner.py:48-177,
cited OPR:line) and `task_registry` need so that they run UNMODIFIED on the fused path.

* `FusedActorCritic` -- an `nn.Module` with the constructor signature of `rsl_rl.modules.ActorCritic` (AC:86-95).  Its parameters are
  views of the flat fp32 buffer the kernels update in place, so `summary(self.alg.actor_critic)` (OPR:78), `.to(device)` (OPR:71),
  `.train()` (OPR:116), `state_dict()` / `load_state_dict()` with the reference's key names (OPR:276-290), `std` (OPR:216) and
  `act_inference` (AC:347-349, used by play.py / get_inference_policy OPR:292-296) behave as the runner expects.
* `install(opr_module)` -- puts `FusedActorCritic` and `FusedPPO` into the namespace OPR:63,72 `eval()`s class names in.
* `make_fused_widowgo1(WidowGo1)` -- returns the `WidowGo1` subclass whose post-physics half is the fused kernel.  legged_gym (and
  through it Isaac Gym) is imported by the caller, never by this package.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib as L
from .actor_critic import FlatActorCritic
from .ppo import FusedPPO


class FusedActorCritic(nn.Module):
    is_recurrent = False

    def __init__(self, num_actor_obs, num_critic_obs, num_actions, actor_hidden_dims=(256, 256, 256), critic_hidden_dims=(256, 256, 256),
                 priv_encoder_dims=(64, 20), activation="elu", init_std=1, **kwargs):
        super().__init__()
        device = kwargs.pop("device", "cuda:0" if torch.cuda.is_available() else "cpu")
        self._ctor = dict(num_actor_obs=num_actor_obs, num_critic_obs=num_critic_obs, num_actions=num_actions, actor_hidden_dims=tuple(actor_hidden_dims),
                          critic_hidden_dims=tuple(critic_hidden_dims), priv_encoder_dims=tuple(priv_encoder_dims), activation=activation,
                          init_std=init_std if not isinstance(init_std, (int, float)) else [[float(init_std)] * num_actions], **kwargs)
        self._attach(FlatActorCritic(device=device, **self._ctor))
        self._ws = None
        self._tmp = None

    def _attach(self, core: FlatActorCritic):
        object.__setattr__(self, "core", core)           # not a sub-module: the flat buffer is the single owner of the values
        for name in list(self._parameters):
            del self._parameters[name]
        for name, view in core.views.items():             # nn.Parameter over a view shares the storage: kernels and torch see the same bytes
            self.register_parameter("p__" + name.replace(".", "__"), nn.Parameter(view, requires_grad=False))

    def __getattr__(self, name):                          # flat / net_cfg / offsets / manifest / hist_range / unflat / num_params ... of the core
        try:
            return super().__getattr__(name)
        except AttributeError:
            core = self.__dict__.get("core")
            if core is not None and hasattr(core, name):
                return getattr(core, name)
            raise

    # ---- what the runner calls ------------------------------------------------------------------------------------------
    def to(self, device=None, *args, **kwargs):           # OPR:71: constructed without a device, then moved
        dev = torch.device(device) if device is not None else self.core.device
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if dev != self.core.device:
            sd = self.core.state_dict()
            core = FlatActorCritic(device=dev, **self._ctor)
            core.load_state_dict(sd)
            self._attach(core)
            self._ws = self._tmp = None
        return self

    def state_dict(self, *args, **kwargs):                # reference key names ("actor.priv_encoder.0.weight", ..., "std")
        return self.core.state_dict()

    def load_state_dict(self, sd, strict=True):
        self.core.load_state_dict(sd, strict)

    @property
    def std(self):
        return self.core.std

    def reset(self, dones=None):
        pass

    def _scratch(self, n):
        lib = L.lib()
        if self._ws is None or self._ws_rows < n:
            nbytes = lib.dwbc_workspace_bytes(C.addressof(self.core.net_cfg), n)
            self._ws, self._ws_rows = torch.zeros(nbytes // 4 + 64, device=self.core.device), n
        na = self.core.num_leg_actions + self.core.num_arm_actions
        if self._tmp is None or self._tmp[0].shape[0] != n:
            z = lambda *s: torch.zeros(*s, device=self.core.device)  # noqa: E731
            self._tmp = [z(n, na), z(n, na), z(n, na), z(n, na), z(n, 2), z(n, 2)]     # eps, actions, mean, sigma, values, log-prob
        return lib

    def act_inference(self, observations, hist_encoding=False):
        """AC:347-349: the action mean, by the actor alone (FlatActorCritic.act_inference: dwbc_policy_mean, the bits of dwbc_policy_act's
        mean)."""
        return self.core.act_inference(observations, hist_encoding)

    def evaluate(self, critic_observations, **kwargs):
        """AC:351-353."""
        obs = critic_observations.contiguous()
        n = obs.shape[0]
        lib = self._scratch(n)
        val = self._tmp[4]
        L.check(lib.dwbc_critic_values(C.addressof(self.core.net_cfg), L.ptr(self.core.flat), L.ptr(obs, torch.float32), obs.stride(0), L.ptr(val), n,
                                       L.ptr(self._ws), L.stream_ptr()), "dwbc_critic_values")
        return val.clone()


def install(opr_module, algorithm_name="FusedPPO", policy_name="FusedActorCritic"):
    """OPR:63 / OPR:72 resolve `runner.policy_class_name` / `runner.algorithm_class_name` with eval() inside
    rsl_rl.runners.on_policy_runner: give that namespace the fused classes.  Then set the two names in the train cfg."""
    setattr(opr_module, policy_name, FusedActorCritic)
    setattr(opr_module, algorithm_name, FusedPPO)
    return dict(policy_class_name=policy_name, algorithm_class_name=algorithm_name)


def make_fused_widowgo1(WidowGo1, gymtorch=None):
    """`class FusedWidowGo1(WidowGo1)`: `step()` (WG:1156-1199), the physics loop, `train.py` and `task_registry` stay the reference's;
    the body of `post_physics_step` after the four gym.refresh_* calls (WG:875-910) is ONE kernel launch.  Register it with
    `task_registry.register("widowGo1", make_fused_widowgo1(WidowGo1, gymtorch), WidowGo1RoughCfg(), WidowGo1RoughCfgPPO())`."""
    from .config import WidowGo1Params
    from .env import FusedWidowGo1Core

    class FusedWidowGo1(WidowGo1):
        def _init_scratch(self):
            super()._init_scratch()                                   # Isaac Gym tensors, URDF-derived tables (WG:498-672)
            p = WidowGo1Params.from_legged_gym(
                self.cfg, num_envs=self.num_envs, dt=self.dt, dof_names=self.dof_names, num_bodies=self.num_bodies, gripper_idx=self.gripper_idx,
                feet_indices=self.feet_indices.tolist(), penalized_contact_indices=self.penalized_contact_indices.tolist(),
                termination_contact_indices=self.termination_contact_indices.tolist(), dof_pos_limits=self.dof_pos_limits.tolist(),
                dof_vel_limits=self.dof_vel_limits.tolist(), torque_limits=self.torque_limits.tolist(), default_dof_pos=self.default_dof_pos.tolist(),
                base_init_state=self.base_init_state.tolist(), reward_scales=self.reward_scales, arm_reward_scales=self.arm_reward_scales)
            self.core = FusedWidowGo1Core(p, self.device)
            self._bind_core()
            st = dict(mass_params=self.mass_params_tensor, friction=self.friction_coeffs_tensor, motor_strength=self.motor_strength,
                      env_origins=self.env_origins, box_env_origins_delta_y=self.box_env_origins_delta_y, traj_timesteps=self.traj_timesteps,
                      traj_total_timesteps=self.traj_total_timesteps)
            if self.cfg.terrain.measure_heights:
                st["height_samples"] = self.height_samples
            self.core.load_state(st)

        def _bind_core(self):
            self.core.bind_sim(root_states=self._root_states, dof_state=self.dof_state, rigid_body_state=self._rigid_body_state,
                               contact_forces=self._contact_forces, force_sensor=self.force_sensor_tensor, torques=self.torques)   # zero-copy views

        def update_command_curriculum(self):                          # WG:678-692: host schedules; the kernel reads the core's copy
            super().update_command_curriculum()
            self.core.update_command_curriculum()

        def post_physics_step(self):
            for f in (self.gym.refresh_actor_root_state_tensor, self.gym.refresh_net_contact_force_tensor,
                      self.gym.refresh_force_sensor_tensor, self.gym.refresh_rigid_body_state_tensor):
                f(self.sim)                                            # WG:870-873 unchanged
            c = self.core
            if c.torques.data_ptr() != self.torques.data_ptr():        # step() rebinds self.torques every sub-step (WG:1178)
                c.bind_sim(torques=self.torques)
            c.actions.copy_(self.actions)                              # the delayed action step() produced (WG:1165-1173)
            c.action_history_buf.copy_(self.action_history_buf)
            c.post_physics_step()                                      # ONE kernel launch
            if c.sim_state_dirty and gymtorch is not None:
                # the reference's whole-tensor sets: resets (WG:787,827) AND push steps (WG:813) -- a push-only step must reach the simulator too
                self.gym.set_dof_state_tensor(self.sim, gymtorch.unwrap_tensor(self.dof_state))
                self.gym.set_actor_root_state_tensor(self.sim, gymtorch.unwrap_tensor(self._root_states))
            self.action_history_buf.copy_(c.action_history_buf)        # zeroed rows of reset envs (WG:735)
            self.episode_length_buf, self.common_step_counter = c.episode_length_buf, c.common_step_counter
            self.obs_buf, self.rew_buf, self.arm_rew_buf, self.reset_buf, self.time_out_buf, self.extras = \
                c.obs_buf, c.rew_buf, c.arm_rew_buf, c.reset_buf, c.time_out_buf, c.extras

    return FusedWidowGo1
