"""CPU: GraphRunner without a GPU.  Its refusals (before any launch), the order of an iteration and the DAgger schedule (OPR:129,
166-169) with the launches stubbed out, the log rows it reads from hand-made device values against the readers they restate
(statistics.mean over rsl_rl's deques, FusedPPO's update() / update_dagger() / update_diagnostics() arithmetic, env.episode_stats()),
and the checkpoint's keys.  The GPU runs are tests/test_gpu_graph_runner.py."""
import collections
import statistics

import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200.config import METRIC_NAMES, CommandCurriculum, WidowGo1Params
from dwbc_b200.env import FusedWidowGo1Core
from dwbc_b200.ppo import FusedPPO
from dwbc_b200.runner import DAGGER_KEY, PPO_KEYS, GraphRunner
from test_oracle_golden import ppo_hp
from test_resume_cpu import make_alg

N, T = 4, 3


class FakeEnv:
    """The host surface of FusedWidowGo1Core the runner touches, with the core's own episode-statistics arithmetic."""
    _fill_episode_extras = FusedWidowGo1Core._fill_episode_extras
    _curriculum_coeffs = FusedWidowGo1Core._curriculum_coeffs
    episode_stats = FusedWidowGo1Core.episode_stats

    def __init__(self, sync_stats=False):
        self.p = WidowGo1Params(num_envs=N, **{k + "_schedule": [0, 6] for k in ("lin_vel_x", "ang_vel_yaw", "tracking_ang_vel_yaw")})
        self.num_envs, self.device, self.sync_stats = N, torch.device("cpu"), sync_stats
        self.sum_names = self.p.sum_slots()
        self._stats = torch.zeros(1 + (len(self.sum_names) + len(METRIC_NAMES) + 3) // 4 * 4)
        self.extras = {"episode": {}}
        self.curriculum = CommandCurriculum(self.p)
        self.obs_buf = torch.zeros(N, 860)
        self.episode_length_buf = torch.zeros(N, dtype=torch.long)
        self.max_episode_length = 1001
        self.events = []

    def update_command_curriculum(self):
        self.curriculum.update()
        self.events.append("curriculum")

    def get_observations(self):
        return self.obs_buf

    def state_dict(self):
        return dict(stats=self._stats.clone(), update_counter=self.curriculum.update_counter)

    def load_state_dict(self, sd):
        self._stats.copy_(sd["stats"])
        self.curriculum.update_counter = sd["update_counter"]


def tracked_alg(track=5, diagnostics=False, **kw):
    ac = make_alg().actor_critic
    alg = FusedPPO(ac, device="cpu", track_episodes=track, diagnostics=diagnostics, **dict(ppo_hp(), **kw))
    alg.init_storage(N, T, [ac.num_obs], [None], [18])
    alg.generator = torch.Generator().manual_seed(3)
    return alg


def launches():
    return L.lib().dwbc_launch_count()


@pytest.mark.parametrize("what", ["world_size", "sync_stats", "no_storage", "mid_rollout", "no_tracker", "log_interval", "save_interval"])
def test_refusals_come_before_any_launch(what):
    alg, env, kw = tracked_alg(track=0 if what == "no_tracker" else 5), FakeEnv(sync_stats=what == "sync_stats"), {}
    if what == "world_size":
        alg.world_size = 2
    elif what == "no_storage":
        alg.storage = None
    elif what == "mid_rollout":
        alg.storage.step = 1
    elif what in ("log_interval", "save_interval"):
        kw = {what: 0}
    n0 = launches()
    with pytest.raises(L.DwbcError):
        GraphRunner(alg, env, **kw)
    for bad in (True, 1.5, -2):
        if what in ("log_interval", "save_interval"):
            with pytest.raises(L.DwbcError):
                GraphRunner(alg, env, **{what: bad})
    assert launches() == n0


def test_learn_refuses_a_state_changed_after_construction():
    alg, env = tracked_alg(), FakeEnv()
    r = GraphRunner(alg, env)
    n0 = launches()
    for change, undo in ((lambda: setattr(env, "sync_stats", True), lambda: setattr(env, "sync_stats", False)),
                         (lambda: setattr(alg.storage, "step", 2), lambda: setattr(alg.storage, "step", 0))):
        change()
        with pytest.raises(L.DwbcError):
            r.learn(1)
        undo()
    assert launches() == n0 and r.current_learning_iteration == 0


def stub_launches(r, events):
    """Replace every launch of an iteration by a record of it; the schedules, the storage and counter move as in FusedPPO."""
    alg = r.alg

    def rollout(obs, hist_encoding):
        events.append(("rollout", hist_encoding))
        alg.storage.step = alg.storage.num_transitions_per_env
        return obs
    r.rollout.run = rollout
    alg.compute_returns = lambda obs: events.append("compute_returns")
    alg._ppo_run = lambda graphed: (events.append(("update", graphed)), alg._fill_hp())[1]
    alg._dagger_run = lambda graphed: events.append(("update_dagger", graphed))
    alg.enforce_min_std = lambda: events.append("enforce_min_std")


@pytest.mark.parametrize("capture", [False, True])
def test_iteration_order_and_dagger_schedule(capture, tmp_path):
    alg, env = tracked_alg(dagger_update_freq=3), FakeEnv()
    saved = []
    r = GraphRunner(alg, env, log_interval=4, save_interval=4, capture=capture,
                    save_path=lambda it: (saved.append(it), str(tmp_path / f"model_{it}.pt"))[1])
    events = env.events
    stub_launches(r, events)
    r.learn(7)
    assert [GraphRunner.dagger_iteration(it, 3) for it in range(7)] == [True, False, False, True, False, False, True]
    per_it = []
    for it in range(7):
        dagger = it % 3 == 0
        per_it += ["curriculum", ("rollout", dagger), "compute_returns"]
        per_it += [("update_dagger", capture)] if dagger else [("update", capture), "enforce_min_std"]
    assert events == per_it
    assert saved == [0, 4, 7] and alg.counter == 7 and r.current_learning_iteration == 7
    rows = r.logs()
    assert [row["iteration"] for row in rows] == list(range(7))
    assert [row["hist_encoding"] for row in rows] == [it % 3 == 0 for it in range(7)]
    assert all((DAGGER_KEY in row) == row["hist_encoding"] and (PPO_KEYS[0] in row) != row["hist_encoding"] for row in rows)
    events.clear()
    r.learn(2)                                                  # continues at iteration 7, a PPO iteration, then 8
    assert [e for e in events if isinstance(e, tuple) and e[0] == "rollout"] == [("rollout", False), ("rollout", False)]
    assert [row["iteration"] for row in r.logs()] == [7, 8] and saved[-1] == 9


def deque_means(appended, cap):
    """rsl_rl's deques (maxlen cap) fed the episodes in order, and OPR.log's statistics.mean over them."""
    d = collections.deque(maxlen=cap)
    d.extend(appended)
    return [statistics.mean(c) for c in zip(*d)] if d else [None, None, None]


def fill_ring(alg, appended):
    """The tracker's ring and position after `appended` episodes, as dwbc_track_episodes leaves them."""
    ring, pos = alg._episodes["ring"], alg._episodes["pos"]
    cap = ring.shape[0]
    ring.zero_()
    for i, e in enumerate(appended):
        ring[i % cap] = torch.tensor(e)
    pos.copy_(torch.tensor([len(appended) % cap, len(appended)]))


def test_rows_equal_the_readers_they_restate():
    """Hand-made device values for six iterations (an empty ring, a partly filled one, one that wrapped more than twice; iterations
    with and without ended episodes): every row equals what the eager readers return on the same values at the same point --
    update()'s / update_dagger()'s endings, statistics.mean over rsl_rl's deques, episode_stats() of a second env fed the same
    statistics, update_diagnostics()."""
    cap = 5
    alg, env, ref = tracked_alg(track=cap, diagnostics=True, dagger_update_freq=3), FakeEnv(), FakeEnv()
    alg.enforce_min_std = lambda: None
    r = GraphRunner(alg, env, log_interval=4)
    g = torch.Generator().manual_seed(9)
    rand = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    episodes = [tuple(float(x) for x in rand(3)) for _ in range(3 * cap + 2)]
    plan = [(0, 0.0), (2, 3.0), (2, 0.0), (cap + 1, 2.0), (3 * cap + 2, 5.0), (3 * cap + 2, 0.0)]      # episodes appended so far, ended
    want = []
    for it, (n_app, ended) in enumerate(plan):
        dagger = it % 3 == 0
        env.update_command_curriculum()
        ref.update_command_curriculum()
        alg._losses.copy_(rand(5).abs() * 7)
        alg.actor_critic.std.copy_(rand(1, 18).abs())
        fill_ring(alg, episodes[:n_app])
        env._stats.copy_(rand(env._stats.numel()).abs())
        env._stats[0] = ended
        ref._stats.copy_(env._stats)
        alg._diag_buffer().copy_(rand(*alg._diag.shape))
        alg._diag_ev.copy_(rand(2))
        row = dict(iteration=it, hist_encoding=dagger)
        if dagger:
            row[DAGGER_KEY] = alg._dagger_finish()
            sched = None
        else:
            result = alg._ppo_finish(alg._fill_hp())
            row.update(zip(PPO_KEYS, result))
            sched = (result[3], result[4], result[6])
        means = deque_means(episodes[:n_app], cap)
        assert [statistics.mean(v) if v else None for v in alg.episode_buffers().values()] == means
        row.update(mean_reward=means[0], mean_arm_reward=means[1], mean_episode_length=means[2])
        row["episode"] = dict(ref.episode_stats())
        row["std"] = alg.actor_critic.std.reshape(-1).tolist()
        row["diagnostics"] = None if dagger else alg.update_diagnostics()
        want.append(row)
        r._snapshot(it, sched)
        assert not env._stats.any()                           # reset as episode_stats() resets it
    entropy, alg.last_entropy = alg.last_entropy, None
    got = r.logs()
    assert got == want
    assert alg.last_entropy == entropy and r.logs() == []
    key = "rew_" + env.sum_names[0]
    assert torch.equal(got[2]["episode"][key], got[1]["episode"][key])          # no episode ended: the previous values carry over
    assert got[2]["episode"]["coeff_lin_vel_x_upper_bound"] != got[1]["episode"]["coeff_lin_vel_x_upper_bound"]


def test_checkpoint_keys_and_load(tmp_path):
    alg, env = tracked_alg(dagger_update_freq=3), FakeEnv()
    r = GraphRunner(alg, env, save_path=lambda it: str(tmp_path / f"model_{it}.pt"))
    stub_launches(r, env.events)
    r.learn(2)
    ck = torch.load(tmp_path / "model_2.pt", weights_only=True)
    assert set(ck) == {"model_state_dict", "optimizer_state_dict", "iter", "infos", "dwbc"}
    assert set(ck["dwbc"]) == {"alg", "env", "iteration", "logs", "episode"}
    assert ck["iter"] == ck["dwbc"]["iteration"] == 2 and ck["infos"] is None
    assert list(ck["model_state_dict"]) == list(alg.actor_critic.state_dict())
    assert [row["iteration"] for row in ck["dwbc"]["logs"]] == [0, 1]             # read for the save, not yet returned by logs()
    from dwbc_b200.runner_compat import FusedActorCritic
    FusedActorCritic(76, 76, 18, actor_hidden_dims=(128,), critic_hidden_dims=(128,), num_priv=24, num_hist=10, num_prop=76,
                     device="cpu").load_state_dict(ck["model_state_dict"])         # strict

    alg2, env2 = tracked_alg(dagger_update_freq=3), FakeEnv()
    alg2.counter = 40
    r2 = GraphRunner(alg2, env2)
    r2.load(str(tmp_path / "model_2.pt"))
    assert r2.current_learning_iteration == 2 and alg2.counter == alg.counter
    assert [row["iteration"] for row in r2.logs()] == [0, 1]
    torch.save({"model_state_dict": {}}, tmp_path / "other.pt")          # OPR.save's file without the 'dwbc' entry
    with pytest.raises(L.DwbcError):
        r2.load(str(tmp_path / "other.pt"))
