"""Shared test helpers: build oracle / kernel env state from the synthetic factories."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import dwbc_b200  # noqa: E402,F401
from dwbc_b200 import synth  # noqa: E402

_DEFAULT_DOF_POS = dwbc_b200.WidowGo1Params().default_dof_pos     # repeated per leg: [0.1, 0.8, -1.5] with the hip sign alternating
ENV_CONFIGS = {
    # default widowGo1 flat config (BASELINE.json configs[1] semantics)
    "flat": dict(),
    # BASELINE.json configs[2]: flat reward set + 187-point height scan on the widowGo1 field (WG:253: 10000 x 600 int16) + terrain curriculum
    "rough": dict(measure_heights=True, tot_rows=10000, tot_cols=600, terrain_curriculum=True),
    # every optional branch: extra reward terms on both channels, termination terms, contact
    # termination, positive-reward clip off, height scan on, terrain curriculum on (LR:421-441)
    "full": dict(
        measure_heights=True, tot_rows=400, tot_cols=600, termination_contact_indices=[2], terrain_curriculum=True,
        reward_scales={
            "action_rate": -0.01, "ang_vel_xy": -0.05, "base_height": -1.0, "collision": -1.0, "dof_acc": -2.5e-7,
            "dof_pos_limits": -10.0, "dof_vel": -1e-3, "dof_vel_limits": -0.1, "energy_square": -6e-5,
            "feet_air_time": 1.0, "feet_contact_forces": -0.01, "foot_contacts_z": -1e-4, "hip_action_l2": -0.01,
            "leg_action_l2": -0.005, "leg_energy": -1e-3, "leg_energy_abs_sum": -1e-3, "leg_energy_sum_abs": -1e-3,
            "lin_vel_z": -2.0, "stand_still": -0.1, "stumble": -0.5, "survive": 0.2, "termination": -2.0,
            "torque_limits": -0.01, "torques": -1e-5, "tracking_ang_vel": 0.5, "tracking_ang_vel_yaw_exp": 0.15,
            "tracking_ang_vel_yaw_l1": 0.1, "tracking_lin_vel": 1.0, "tracking_lin_vel_x_exp": 0.2,
            "tracking_lin_vel_x_l1": 0.5, "tracking_lin_vel_y_l2": -0.1, "tracking_lin_vel_z_l2": -0.1},
        arm_reward_scales={
            "arm_energy_abs_sum": -0.004, "termination": -1.0, "tracking_ee_cart": 0.3, "tracking_ee_orn": 0.1,
            "tracking_ee_orn_ry": 0.1, "tracking_ee_sphere": 0.55}),
    # The configs below each set the fields of one branch no shipped config takes (the kernels read them from DwbcEnvCfg / the device
    # step record); everything else stays at the defaults of `flat`.
    # cart goals (WG:1360-1366, command_mode): termination signs and observation goal columns read the cart goal; non-zero orientation
    # deltas whose yaw part d + yaw leaves (-pi, pi], so the wrap of the goal orientation runs (WG:1307-1313)
    "cart": dict(
        command_mode="cart", final_delta_orn=[[-0.6, 0.6], [-0.4, 0.8], [-2.6, 2.6]],
        arm_reward_scales={"arm_energy_abs_sum": -0.004, "tracking_ee_cart": 0.55, "tracking_ee_orn": 0.1, "tracking_ee_orn_ry": 0.1}),
    # only_positive_rewards and termination on both channels (WG:170-205): mostly negative leg scales, so the channel sum is often
    # clipped before the termination term is added; the shared `termination` sum slot takes both channels' additions
    "positive": dict(
        only_positive_rewards=True,
        reward_scales={"energy_square": -6e-5, "foot_contacts_z": -1e-4, "hip_action_l2": -0.02, "survive": 0.05, "termination": -2.0,
                       "torques": -1e-4, "dof_vel": -2e-3, "tracking_ang_vel_yaw_exp": 0.15, "tracking_lin_vel_x_l1": 0.5},
        arm_reward_scales={"arm_energy_abs_sum": -0.004, "termination": -1.0, "tracking_ee_sphere": 0.55}),
    # EE-goal search (WG:1316-1342): a collision box and an underground limit that reject most paths, so the winning try takes every
    # index 0..9 and some searches use up all ten tries; num_collision_check_samples is set per case (goals_case)
    "goals": dict(underground_limit=-0.1, collision_upper_limits=[0.45, 0.3, 0.1], collision_lower_limits=[-0.3, -0.3, -0.6]),
    # no DOF reordering (WG:1003-1048) and no push (WG:804-814, 934); 8 penalised and 3 termination contact bodies; per-joint distinct
    # defaults and limits, read by the reset, the observation and the DOF reward terms
    "raw": dict(
        reorder_dofs=False, push_robots=False,
        penalized_contact_indices=[1, 2, 3, 4, 6, 7, 8, 10], termination_contact_indices=[11, 14, 19],
        default_dof_pos=[round(d + 0.013 * (i + 1), 3) for i, d in enumerate(_DEFAULT_DOF_POS)],
        dof_pos_limits=[[round(d + 0.013 * (i + 1) - 0.3 - 0.02 * i, 3), round(d + 0.013 * (i + 1) + 0.25 + 0.015 * i, 3)]
                        for i, d in enumerate(_DEFAULT_DOF_POS)],
        dof_vel_limits=[round(1.0 + 0.17 * i, 3) for i in range(20)],
        torque_limits=[round(3.0 + 0.9 * i, 3) for i in range(20)], soft_torque_limit=0.85,
        reward_scales={"collision": -1.0, "dof_pos_limits": -10.0, "dof_vel_limits": -0.1, "energy_square": -6e-5, "foot_contacts_z": -1e-4,
                       "hip_action_l2": -0.01, "stand_still": -0.1, "survive": 0.2, "termination": -2.0, "torque_limits": -0.01,
                       "tracking_ang_vel_yaw_exp": 0.15, "tracking_lin_vel_x_l1": 0.5}),
    # action delay FIFO (WG:1162-1173) with a binding clip_actions; action_delay is set per case (delay_case)
    "delay": dict(clip_actions=0.5),
}
COLLISION_SAMPLES = (0, 1, 3, 10, 11, 16)       # 32 / S tries per round of the kernels' goal search: 32, 32, 10, 3, 2, 2
ACTION_DELAYS = (0, 1, 6)                        # action_hist_len 2, 3, 8


def goals_case(S):
    return dict(ENV_CONFIGS["goals"], num_collision_check_samples=S)


def delay_case(d):
    return dict(ENV_CONFIGS["delay"], action_delay=d, action_hist_len=d + 2)


# every config-branch case by name: the new configs, `goals` once per sample count, `delay` once per delay
BRANCH_CASES = dict(
    [(k, ENV_CONFIGS[k]) for k in ("cart", "positive", "raw")] + [(f"goals-{s}", goals_case(s)) for s in COLLISION_SAMPLES] +
    [(f"delay-{d}", delay_case(d)) for d in ACTION_DELAYS])


def make_params(name, num_envs):
    return dwbc_b200.WidowGo1Params(num_envs=num_envs, **ENV_CONFIGS[name])


def runtime(p, counter=1):
    """Curriculum outputs after `counter` calls of update_command_curriculum (WG:678-692)."""
    cur = dwbc_b200.CommandCurriculum(p)
    for _ in range(counter):
        cur.update()
    return SimpleNamespace(lin_vel_x=cur.lin_vel_x_ranges, ang_vel_yaw=cur.ang_vel_yaw_ranges,
                           goal_l=cur.goal_ee_l_ranges, goal_p=cur.goal_ee_p_ranges, goal_y=cur.goal_ee_y_ranges,
                           leg_scales=cur.reward_scales, arm_scales=cur.arm_reward_scales)


def initial(p, seed):
    st = synth.initial_env_state(p, seed)
    st.update(synth.sim_state(p, seed, 0))
    if p.measure_heights:
        st["height_samples"] = synth.height_field(p, seed)
    return st


def sim_state(p, seed, t, env_origins=None, **kw):
    """synth.sim_state, with the robot placed RELATIVE to its current env origin when the terrain curriculum is on
    (LR:430 measures the distance walked from the origin: absolute +-5 m positions would make every reset a promotion).
    `env_origins` = the [N,3] origins before the step (numpy / tensor), i.e. state the caller carries."""
    sim = synth.sim_state(p, seed, t, **kw)
    if p.terrain_curriculum and env_origins is not None:
        org = env_origins.detach().cpu().numpy() if isinstance(env_origins, torch.Tensor) else np.asarray(env_origins)
        sim["root_states"][:, 0, 0:2] += org[:, 0:2].astype(np.float32)
    return sim


def oracle_state(p, st):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).clone()  # noqa: E731
    N = p.num_envs
    s = SimpleNamespace(
        root_states_full=T(st["root_states"]), dof_state=T(st["dof_state"]), rigid_body_state=T(st["rigid_body_state"]),
        contact_forces_full=T(st["contact_forces"]), force_sensor=T(st["force_sensor"]), torques=T(st["torques"]),
        action_history_buf=T(st["action_history_buf"]),
        base_lin_vel=torch.zeros(N, 3), base_ang_vel=torch.zeros(N, 3), base_yaw_euler=torch.zeros(N, 3),
        base_yaw_quat=torch.zeros(N, 4), mass_params=T(st["mass_params"]), friction=T(st["friction"]),
        motor_strength=T(st["motor_strength"]))
    for k in ("commands", "goal_timer", "traj_timesteps", "traj_total_timesteps", "ee_start_sphere", "ee_goal_sphere",
              "ee_goal_cart", "curr_ee_goal_sphere", "curr_ee_goal_cart", "ee_goal_delta_orn_euler",
              "ee_goal_orn_euler", "obs_history_buf", "last_actions", "last_dof_vel", "last_root_vel", "feet_air_time",
              "last_contacts", "env_origins", "box_env_origins_delta_y", "episode_length_buf", "terrain_levels",
              "terrain_types", "terrain_origins"):
        setattr(s, k, T(st[k]))
    s.actions = s.action_history_buf[:, -(p.action_delay + 1)].clone()
    if "height_samples" in st:
        s.height_samples = T(st["height_samples"])
    return s


def load_sim_into_oracle(o, p, sim):
    s = o.s
    s.root_states_full.copy_(torch.from_numpy(sim["root_states"]))
    s.dof_state.copy_(torch.from_numpy(sim["dof_state"]))
    s.rigid_body_state.copy_(torch.from_numpy(sim["rigid_body_state"]))
    s.contact_forces_full.copy_(torch.from_numpy(sim["contact_forces"]))
    s.force_sensor.copy_(torch.from_numpy(sim["force_sensor"]))
    s.torques = torch.from_numpy(sim["torques"]).clone()
    a = torch.from_numpy(sim["policy_actions"])[:, p.raisim2ig(p.num_actions)]
    a = torch.clip(a, -p.clip_actions, p.clip_actions)                                   # WG:1163
    s.action_history_buf = torch.cat([s.action_history_buf[:, 1:], a[:, None, :]], dim=1)  # WG:1166
    s.actions = s.action_history_buf[:, -(p.action_delay + 1)].clone()                    # WG:1167-1168
