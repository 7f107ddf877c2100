"""GPU: the episode tracker of FusedPPO(track_episodes=C) (dwbc_track_episodes) computes what OnPolicyRunner's per-step bookkeeping
(OPR:140-154) computes, bit for bit.
  * The kernel against the restatement of tests/test_episode_tracking_cpu.py over 60 steps, at 1 to 40 000 envs, C = 1 to 1000, done
    rates 0, 2 % and 100 % (a step that finishes more than C episodes), dones as bool and as uint8.
  * In the training workload (direct-to-storage transitions, time-outs, nonzero values): the tracker follows the un-bootstrapped
    env rewards, not the bootstrapped storage rows.
  * A captured rollout (RolloutGraph) tracks what the eager loop tracks, over two PPO and one DAgger iteration, with no library launch
    during a replay; a resumed run tracks what a run that never stopped tracks; track_episodes=0 launches and saves what a FusedPPO
    built without it does.
  * The unmodified runner (when baseline/_ref holds the reference): its rewbuffer / arm_rewbuffer / lenbuffer deques equal
    episode_buffers() after every iteration."""
import os
import sys

import pytest
import torch

import test_gpu_resume as R
from dwbc_b200 import _lib as L
from dwbc_b200.ppo import FusedPPO
from test_episode_tracking_cpu import KEYS, Restatement, stream
from test_gpu_cuda_graphs import ReplayLaunches, assert_bitwise, run_workload

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def tracking(monkeypatch, cap, made=None):
    """Every FusedPPO the workload builders construct from now on gets track_episodes=cap (and is appended to `made`)."""
    from dwbc_b200 import ppo

    class Tracking(FusedPPO):
        def __init__(self, *a, **k):
            super().__init__(*a, track_episodes=cap, **k)
            if made is not None:
                made.append(self)
    monkeypatch.setattr(ppo, "FusedPPO", Tracking)


def ring_buffers(ring, pos, cap):
    """The deques the ring holds, oldest first (dwbc.h: oldest at slot (next - min(total, C)) mod C)."""
    ring, (nxt, total) = ring.cpu(), pos.tolist()
    n = min(total, cap)
    rows = ring[[(nxt - n + i) % cap for i in range(n)]]
    return {k: rows[:, c].tolist() for c, k in enumerate(KEYS)}


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8])
@pytest.mark.parametrize("rate", [0.0, 0.02, 1.0])
@pytest.mark.parametrize("cap", [1, 100, 1000])
@pytest.mark.parametrize("n", [1, 33, 4096, 40000])
def test_kernel_equals_the_restatement(n, cap, rate, dtype):
    lib = L.lib()
    ref = Restatement(n, cap)
    running, ring = torch.zeros(n, 3, device=DEV), torch.zeros(cap, 3, device=DEV)
    pos = torch.zeros(2, dtype=torch.int64, device=DEV)
    appended = 0
    for rew, arm, dones in stream(n, 60, rate, 7 * n + cap, dtype):
        r, a, d = rew.to(DEV), arm.to(DEV), dones.to(DEV)
        L.check(lib.dwbc_track_episodes(L.ptr(r), L.ptr(a), L.ptr(d), n, L.ptr(running), L.ptr(ring), L.ptr(pos), cap, L.stream_ptr()),
                "dwbc_track_episodes")
        ref.step(rew, arm, dones)
        appended += int(dones.bool().sum())
    assert torch.equal(running.cpu(), ref.running)
    assert int(pos[1]) == appended
    assert ring_buffers(ring, pos, cap) == ref.buffers()
    assert appended == {0.0: 0, 1.0: 60 * n}.get(rate, appended) and (n < 4096 or rate == 0.0 or appended > cap)


def test_tracks_the_env_rewards_not_the_storage_rows(monkeypatch):
    """Eager rollout with the post-physics kernel writing the transition rows; episode lengths start near the limit, so that envs time
    out and the storage rows carry gamma * value bootstraps the tracker must not see."""
    tracking(monkeypatch, 100)
    w = R.build(10, 4096, "flat", "tf32x3", False, 0)
    env, alg, s = w.env, w.alg, w.alg.storage
    n, limit = s.num_envs, int(env.max_episode_length)
    g = torch.Generator().manual_seed(5)
    env.episode_length_buf.copy_(torch.randint(limit - 2 * R.T, limit, (n,), generator=g).to(env.episode_length_buf))
    ref = Restatement(n, 100)
    obs, bootstrapped = s.obs_row(0), 0
    for t in range(R.T):
        actions = alg.act(obs, obs)
        env.bind_sim(**w.pool[t])
        env.set_obs_target(s.obs_row(t + 1))
        env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
        env.pre_physics_step(actions)
        env.post_physics_step()
        obs = env.obs_buf
        alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
        assert env.extras["dwbc_stored_rows"] == (s.rewards[t].data_ptr(), s.dones[t].data_ptr())    # the kernel stored the row
        ref.step(env.rew_buf.cpu(), env.arm_rew_buf.cpu(), env.reset_buf.cpu())
        to = env.time_out_buf.cpu()
        bootstrapped += int((s.rewards[t].cpu() != torch.stack([env.rew_buf, env.arm_rew_buf], 1).cpu())[to].any(1).sum())
    assert bootstrapped > 0                                   # time-outs with nonzero values: the storage rows differ from the rewards
    assert torch.equal(alg._episodes["running"].cpu(), ref.running)
    got = alg.episode_buffers()
    assert got == ref.buffers() and len(got["lenbuffer"]) == 100
    R.free(w)


def test_captured_rollouts_track_what_the_eager_loop_tracks(monkeypatch):
    out = {}
    for graphs in (False, True):
        made = []
        tracking(monkeypatch, 1000, made)
        counter = ReplayLaunches(monkeypatch) if graphs else None
        state = run_workload("tf32x3", graphs, False)
        (alg,) = made
        if graphs:
            assert counter.replays == 6 and counter.moved == 0, (counter.replays, counter.moved)
        bufs = alg.episode_buffers()
        state.update({f"tracker.{k}": v.clone() for k, v in alg._episodes.items()})
        state.update({f"buffer.{k}": torch.tensor(v, dtype=torch.float64) for k, v in bufs.items()})
        out[graphs] = state
        del alg, made
    assert 0 < len(out[False]["buffer.lenbuffer"]) and int(out[False]["tracker.pos"][1]) > 0
    assert_bitwise(out[False], out[True])


@pytest.mark.parametrize("graphs_before,graphs_after", [(False, False), (True, True)])
def test_resumed_run_tracks_what_the_straight_run_tracks(graphs_before, graphs_after, monkeypatch, tmp_path):
    tracking(monkeypatch, 300)
    w = R.build(10, 4096, "flat", "tf32x3", False, 0)
    R.set_graphs(w, graphs_before)
    for dagger in (False, True, False, True):
        R.iteration(w, dagger)
    straight = dict(R.end_state(w), **{f"tracker.{k}": v.clone() for k, v in w.alg._episodes.items()})
    straight_bufs = w.alg.episode_buffers()
    R.free(w)

    w = R.build(10, 4096, "flat", "tf32x3", False, 0)
    R.set_graphs(w, graphs_before)
    for dagger in (False, True):
        R.iteration(w, dagger)
    R.save(w, tmp_path / "ckpt.pt")
    R.free(w)
    w = R.build(10, 4096, "flat", "tf32x3", False, 1, height_field=False)
    R.load(w, torch.load(tmp_path / "ckpt.pt"))
    R.set_graphs(w, graphs_after)
    for dagger in (False, True):
        R.iteration(w, dagger)
    resumed = dict(R.end_state(w), **{f"tracker.{k}": v.clone() for k, v in w.alg._episodes.items()})
    resumed_bufs = w.alg.episode_buffers()
    R.free(w)
    assert len(straight_bufs["lenbuffer"]) > 0 and resumed_bufs == straight_bufs
    assert_bitwise(straight, resumed)


def test_off_launches_and_saves_what_a_ppo_without_it_does(monkeypatch):
    def one_iteration():
        w = R.build(10, 1024, "flat", "tf32x3", False, 0)
        n0 = L.lib().dwbc_launch_count()
        R.iteration(w, False)
        torch.cuda.synchronize()
        launches, keys, tensors = L.lib().dwbc_launch_count() - n0, set(w.alg.state_dict()), set(R._tensors("alg", w.alg))
        R.free(w)
        return launches, keys, tensors
    plain = one_iteration()
    tracking(monkeypatch, 0)
    off = one_iteration()
    tracking(monkeypatch, 100)
    on = one_iteration()
    assert off == plain
    assert on[0] == plain[0] + R.T and on[1] == plain[1] | {"episodes"}


REF = os.path.join(ROOT, "baseline", "_ref")


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "rsl_rl")), reason="needs the unmodified rsl_rl: baseline/install_reference.sh <checkout of the reference>")
def test_unmodified_runner_deques_equal_the_episode_buffers(tmp_path):
    import json
    for pth in (REF, os.path.join(ROOT, "tests", "fakes")):
        if pth not in sys.path:
            sys.path.insert(0, pth)
    import rsl_rl.runners.on_policy_runner as opr
    from dwbc_b200 import runner_compat as RC
    from test_gpu_runner import SyntheticWidowGo1
    cfg = json.load(open(os.path.join(ROOT, "baseline", "widowgo1_train_cfg.json")))
    names = RC.install(opr)
    train_cfg = dict(policy=dict(cfg["policy"]),
                     algorithm=dict(cfg["algorithm"], num_learning_epochs=2, num_mini_batches=2, precision="tf32x3", track_episodes=100),
                     runner=dict(cfg["runner"], num_steps_per_env=24, save_interval=100, **names))
    env = SyntheticWidowGo1(256, DEV)
    runner = opr.OnPolicyRunner(env, train_cfg, log_dir=str(tmp_path), device=DEV)
    seen = []
    log = runner.log

    def checked_log(locs, *a, **k):
        bufs = runner.alg.episode_buffers()
        seen.append({k_: list(locs[k_]) for k_ in KEYS if k_ in locs})
        assert seen[-1].keys() == set(KEYS), sorted(k_ for k_ in locs if k_.endswith("buffer"))
        for k_ in KEYS:
            assert seen[-1][k_] == bufs[k_], k_
        return log(locs, *a, **k)
    runner.log = checked_log
    runner.learn(3, init_at_random_ep_len=True)
    assert len(seen) == 3 and len(seen[-1]["lenbuffer"]) > 0
