"""GPU parity of the fused post-physics kernel (through the C ABI) against the golden vectors
recorded from the unmodified reference and against the CPU oracle."""
import os

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import synth
from oracle import env_oracle as EO

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
FTOL = dict(rtol=2e-5, atol=2e-6)


def make_core(p, st, **kw):
    from dwbc_b200.env import FusedWidowGo1Core
    core = FusedWidowGo1Core(p, "cuda:0", state=st, **kw)
    core.update_command_curriculum()
    return core


def load_sim(core, p, sim):
    dev = core.device
    core._root_states.copy_(torch.from_numpy(sim["root_states"]).to(dev))
    core.dof_state.copy_(torch.from_numpy(sim["dof_state"]).to(dev))
    core._rigid_body_state.copy_(torch.from_numpy(sim["rigid_body_state"]).to(dev))
    core._contact_forces.copy_(torch.from_numpy(sim["contact_forces"]).to(dev))
    core.force_sensor_tensor.copy_(torch.from_numpy(sim["force_sensor"]).to(dev))
    core.torques.copy_(torch.from_numpy(sim["torques"]).to(dev))
    core.pre_physics_step(torch.from_numpy(sim["policy_actions"]).to(dev))


@pytest.mark.parametrize("name", ["flat", "full"])
def test_env_step_matches_reference_golden(name, generic_kernel=False):
    g = np.load(os.path.join(G, f"env_{name}.npz"))
    N, steps, seed, counter0 = [int(x) for x in g["meta"]]
    p = E.make_params(name, N)
    core = make_core(p, E.initial(p, seed), generic_kernel=generic_kernel)
    core.common_step_counter = counter0
    for t in range(1, steps + 1):
        i = t - 1
        load_sim(core, p, E.sim_state(p, seed, t, g["env_origins_pre"][i]))
        core.post_physics_step(torch.from_numpy(synth.rand_table(p, seed, t)).cuda())
        np.testing.assert_array_equal(core.reset_buf.cpu().numpy(), g["reset"][i], err_msg=f"reset step {t}")
        np.testing.assert_array_equal(core.time_out_buf.cpu().numpy(), g["time_out"][i])
        np.testing.assert_array_equal(core.episode_length_buf.cpu().numpy(), g["ep_len"][i])
        np.testing.assert_allclose(core.obs_buf[:, :100].cpu().numpy(), g["obs100"][i], **FTOL, err_msg=f"obs step {t}")
        np.testing.assert_allclose(core.rew_buf.cpu().numpy(), g["rew"][i], **FTOL)
        np.testing.assert_allclose(core.arm_rew_buf.cpu().numpy(), g["arm_rew"][i], **FTOL)
        np.testing.assert_allclose(core.commands.cpu().numpy(), g["commands"][i], **FTOL)
        np.testing.assert_allclose(core.ee_goal_sphere.cpu().numpy(), g["ee_goal_sphere"][i], **FTOL)
        np.testing.assert_array_equal(core.goal_timer.cpu().numpy(), g["goal_timer"][i])
        if p.measure_heights:
            np.testing.assert_allclose(core.measured_heights.cpu().numpy(), g["heights"][i], rtol=1e-6, atol=1e-7)
            np.testing.assert_allclose(core.heights_obs.cpu().numpy(), g["heights_obs"][i], rtol=1e-6, atol=1e-6)   # LR:221-223
        if p.terrain_curriculum:                                                          # LR:421-441 (SURVEY row a21)
            np.testing.assert_array_equal(core.terrain_levels.cpu().numpy(), g["terrain_levels"][i], err_msg=f"terrain level step {t}")
            np.testing.assert_array_equal(core.env_origins.cpu().numpy(), g["env_origins"][i])
        if g["reset"][i].sum():
            ep = core.extras["episode"]
            got = np.array([float(ep[k]) for k in g["stat_names"]], np.float32)
            np.testing.assert_allclose(got, g["ep_stats"][i], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(core.obs_buf.cpu().numpy(), g["final_obs"], **FTOL)
    np.testing.assert_allclose(core.obs_history_buf.cpu().numpy(), g["final_hist"], **FTOL)
    np.testing.assert_allclose(core._root_states.cpu().numpy(), g["final_root"], **FTOL)
    np.testing.assert_allclose(core.dof_state.cpu().numpy(), g["final_dof"], **FTOL)
    np.testing.assert_allclose(core.action_history_buf.cpu().numpy(), g["final_ahist"], **FTOL)
    sums = np.stack([core.episode_sums[k].cpu().numpy() for k in g["sum_names"]])
    np.testing.assert_allclose(sums, g["final_sums"], rtol=1e-4, atol=1e-6)
    from dwbc_b200.config import METRIC_NAMES
    mets = np.stack([core.episode_metric_sums[k].cpu().numpy() for k in METRIC_NAMES])
    np.testing.assert_allclose(mets, g["final_metrics"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name,N", [("flat", 4096), ("full", 1024)])
def test_env_step_matches_oracle_full_size(name, N):
    """BASELINE.json configs[1]/[2] sizes: every state tensor against the CPU oracle, 6 steps."""
    seed = 11
    p = E.make_params(name, N)
    st = E.initial(p, seed)
    core = make_core(p, st)
    orc = EO.EnvOracle(p, E.oracle_state(p, st))
    rt = E.runtime(p)
    core.common_step_counter = orc.common_step_counter = 146
    mism = 0
    for t in range(1, 7):
        sim = E.sim_state(p, seed, t, orc.s.env_origins)
        load_sim(core, p, sim)
        E.load_sim_into_oracle(orc, p, sim)
        tab = torch.from_numpy(synth.rand_table(p, seed, t))
        obs, rew, arew, rst, _ = orc.post_physics_step(tab, rt)
        core.post_physics_step(tab.cuda())
        same = core.reset_buf.cpu() == rst
        mism += int((~same).sum())
        assert mism == 0, f"{mism} discrete reset decisions differ at step {t}"
        np.testing.assert_allclose(core.obs_buf.cpu().numpy(), obs.numpy(), **FTOL)
        np.testing.assert_allclose(core.rew_buf.cpu().numpy(), rew.numpy(), **FTOL)
        np.testing.assert_allclose(core.arm_rew_buf.cpu().numpy(), arew.numpy(), **FTOL)
        for k in ("commands", "goal_timer", "ee_start_sphere", "ee_goal_sphere", "ee_goal_cart", "curr_ee_goal_sphere",
                  "curr_ee_goal_cart", "ee_goal_orn_euler", "base_lin_vel", "base_ang_vel", "base_yaw_quat", "last_root_vel",
                  "last_actions", "last_dof_vel", "feet_air_time"):
            np.testing.assert_allclose(getattr(core, k).cpu().numpy(), getattr(orc.s, k).numpy(), **FTOL, err_msg=k)
        np.testing.assert_allclose(core.obs_history_buf.cpu().numpy(), orc.s.obs_history_buf.numpy(), **FTOL)
        np.testing.assert_allclose(core._root_states.cpu().numpy(), orc.s.root_states_full.numpy(), **FTOL)
        np.testing.assert_allclose(core.dof_state.cpu().numpy(), orc.s.dof_state.numpy(), **FTOL)
        np.testing.assert_array_equal(core.episode_length_buf.cpu().numpy(), orc.s.episode_length_buf.numpy())
        if p.measure_heights:
            np.testing.assert_allclose(core.measured_heights.cpu().numpy(), orc.measured_heights.numpy(), rtol=1e-6, atol=1e-7)
            np.testing.assert_allclose(core.heights_obs.cpu().numpy(),
                                       EO.heights_obs(orc.root[:, 2], orc.measured_heights, p.obs_scale_height).numpy(), rtol=1e-6, atol=1e-6)
        if p.terrain_curriculum:
            np.testing.assert_array_equal(core.terrain_levels.cpu().numpy(), orc.s.terrain_levels.numpy())
            np.testing.assert_array_equal(core.env_origins.cpu().numpy(), orc.s.env_origins.numpy())


def test_philox_mode_equals_table_mode():
    """In-kernel Philox draws == table mode fed with dwbc_fill_uniform of the same (seed, step)."""
    seed, N = 5, 512
    p = E.make_params("flat", N)
    st = E.initial(p, seed)
    a, b = make_core(p, st, seed=1234), make_core(p, st, seed=1234)
    a.common_step_counter = b.common_step_counter = 147
    for t in range(1, 6):
        sim = synth.sim_state(p, seed, t)
        load_sim(a, p, sim)
        load_sim(b, p, sim)
        tab = b.fill_uniform(b.common_step_counter + 1)
        assert float(tab.min()) >= 0.0 and float(tab.max()) < 1.0 and abs(float(tab.mean()) - 0.5) < 0.01
        a.post_physics_step()
        b.post_physics_step(tab)
        for k in ("obs_buf", "rew_buf", "reset_buf", "_goal_state", "_derived_state", "_root_states", "dof_state", "_hist"):
            assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert int(a.reset_buf.sum()) >= 0


def test_obs_written_directly_into_storage_row_and_structure():
    """obs target redirection (SURVEY f2) + size-independent structure of the observation row:
    obs[:,100:] is the previous history; new history = shift/append (or fill after a reset)."""
    seed, N = 9, 4096
    p = E.make_params("flat", N)
    core = make_core(p, E.initial(p, seed))
    store = torch.zeros(3, N, p.num_obs, device="cuda")
    for t in range(1, 3):
        load_sim(core, p, synth.sim_state(p, seed, t))
        prev_hist = core.obs_history_buf.clone()
        core.set_obs_target(store[t])
        core.post_physics_step()
        obs = store[t]
        rst = core.reset_buf
        keep = ~rst
        assert torch.equal(obs[keep][:, 100:], torch.clip(prev_hist[keep].flatten(1), -100, 100))
        assert float(obs[rst][:, 100:].abs().max()) == 0.0 if int(rst.sum()) else True
        prop = obs[:, :76]
        fill = core.episode_length_buf <= 1
        h = core.obs_history_buf
        assert torch.equal(h[:, -1], prop) or torch.allclose(h[:, -1], prop)
        assert torch.equal(h[~fill][:, :-1], prev_hist[~fill][:, 1:])
        assert torch.equal(h[fill], prop[fill][:, None, :].expand(-1, p.history_len, -1))
        assert float(obs.abs().max()) <= 100.0


def test_transition_written_directly_into_storage_rows():
    """SURVEY f2: with set_transition_target the post-physics kernel performs PPO.process_env_step's reward path (PPO:130-134) and the dones
    store (RS:102) itself; bit-identical to the separate dwbc_store_rewards launch, and FusedPPO.process_env_step recognises the rows."""
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    seed, N, T = 13, 2048, 3
    p = E.make_params("flat", N)
    st = E.initial(p, seed)
    a, b = make_core(p, st, seed=5), make_core(p, st, seed=5)
    a.common_step_counter = b.common_step_counter = 148
    algs = []
    for _ in range(2):
        alg = FusedPPO(FlatActorCritic(device="cuda:0", seed=0, num_priv=24, num_hist=10, num_prop=76), device="cuda:0", gamma=0.99)
        alg.init_storage(N, T, [p.num_obs], [None], [p.num_actions])
        alg.storage.values.normal_(generator=torch.Generator(device="cuda").manual_seed(3))
        algs.append(alg)
    n_timeout = n_done = 0
    for t in range(T):
        sim = synth.sim_state(p, seed, t + 1)
        load_sim(a, p, sim)
        load_sim(b, p, sim)
        sa, sb = algs[0].storage, algs[1].storage
        b.set_transition_target(sb.values[t], sb.rewards[t], sb.dones[t], 0.99)
        a.post_physics_step()
        b.post_physics_step()
        n0 = int(a._lib.dwbc_launch_count())
        algs[0].process_env_step(a.rew_buf, a.arm_rew_buf, a.reset_buf, a.extras)
        n1 = int(a._lib.dwbc_launch_count())
        algs[1].process_env_step(b.rew_buf, b.arm_rew_buf, b.reset_buf, b.extras)
        assert n1 - n0 == 1 and int(a._lib.dwbc_launch_count()) == n1          # the second call launched nothing
        assert torch.equal(sa.rewards[t], sb.rewards[t]) and torch.equal(sa.dones[t], sb.dones[t])
        # the bootstrap changed the rows of the timed-out envs (gamma * values, PPO:133-134) and no other row
        to, raw = a.time_out_buf, torch.stack([a.rew_buf, a.arm_rew_buf], dim=-1)
        assert torch.equal(sb.rewards[t][~to], raw[~to])
        assert bool((sb.rewards[t][to] != raw[to]).all(dim=-1).all())
        torch.testing.assert_close(sb.rewards[t][to], raw[to] + 0.99 * sb.values[t][to], rtol=1e-6, atol=1e-6)
        n_timeout += int(to.sum())
        n_done += int(sb.dones[t].sum())
    assert float(algs[0].storage.rewards.abs().sum()) > 0
    assert n_timeout > 0 and n_done > n_timeout, (n_timeout, n_done)          # time-outs and terminations both occurred


@pytest.mark.gpu
def test_torque_controller_matches_reference_golden():
    """dwbc_compute_torques (WG:1262-1295) against the golden vectors of the unmodified reference: exact fp32 arithmetic (the kernel is
    built without FMA contraction); the one wrapped column may differ by an ulp of the angle times p_gain (stated tolerance 5e-5)."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "torques.npz"))
    N = int(g["meta"][0])
    p = E.make_params("flat", N)
    from dwbc_b200.env import FusedWidowGo1Core
    env = FusedWidowGo1Core(p, "cuda:0", state=E.initial(p, 3))
    ds = torch.stack([torch.from_numpy(g["dof_pos"]), torch.from_numpy(g["dof_vel"])], dim=-1).reshape(N * p.num_dofs, 2)
    env.dof_state.copy_(ds.cuda())
    env.motor_strength.copy_(torch.from_numpy(g["motor"]).cuda())
    out = env.compute_torques(torch.from_numpy(g["actions"]).cuda()).cpu().numpy()
    np.testing.assert_allclose(out, g["torques"], rtol=0, atol=5e-5)
    wrap = p.num_actions - 8
    cols = [j for j in range(p.num_dofs) if j != wrap]
    np.testing.assert_array_equal(out[:, cols], g["torques"][:, cols])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["flat", "full"])
def test_general_fallback_kernel_matches_reference_golden(name):
    """`env_step_kernel` (warp per env; any N / n_dof / unaligned buffers) is what runs when the 32-envs-per-CTA TMA kernel does not
    apply; `DwbcStepArgs.generic_kernel` forces it on the golden case."""
    test_env_step_matches_reference_golden(name, generic_kernel=True)
