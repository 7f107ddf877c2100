"""CPU: GraphRunner's scheduled evaluation and throughput figures without a GPU.  The refusals (before any launch), which iterations
evaluate (it % eval_interval == 0, also in runs that start at a resumed iteration) and in what order a mode's run is restored and run,
the eval rows read from hand-made trackers and statistics blocks against rsl_rl's deques and episode_stats() (empty, partly filled and
wrapped rings; one mode and both), the timing fields from hand-made event times, and the checkpoint's keys with and without evaluation
and the refusals to load one into the other.  The GPU runs are tests/test_gpu_graph_runner_eval.py."""
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200.runner import EVAL_MODES, TIMING_KEYS, GraphRunner
from test_graph_runner_cpu import N, T, FakeEnv, deque_means, fill_ring, launches, stub_launches, tracked_alg


class FakeEvalEnv(FakeEnv):
    """FakeEnv with the shape EvalGraph checks against the policy; it records each restore of a snapshot."""

    def __init__(self, sync_stats=False, num_obs=860):
        super().__init__(sync_stats)
        self.num_obs, self.num_actions = num_obs, 18

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        self.events.append("restore")


def make(modes=EVAL_MODES, interval=2, cap=5, ev_env=None, **kw):
    alg, env, ev_env = tracked_alg(dagger_update_freq=3), FakeEnv(), ev_env or FakeEvalEnv()
    r = GraphRunner(alg, env, eval_env=ev_env, eval_interval=interval, eval_steps=4, eval_track_episodes=cap, eval_modes=modes, **kw)
    return r, env, ev_env


def stub_evals(r, events, on_run=None):
    """Replace each mode's EvalGraph run by a record of it (and `on_run(mode)`, which may fill the tracker and statistics)."""
    for m, ev in r._evals.items():
        def run(obs, m=m):
            events.append(("eval", m))
            if on_run is not None:
                on_run(m)
            return obs
        ev.run = run


@pytest.mark.parametrize("what", ["same_core", "sync_stats", "steps_odd", "steps_zero", "steps_none", "interval_zero", "interval_none",
                                  "track_zero", "mode_unknown", "modes_empty", "modes_str", "mismatch"])
def test_eval_refusals_come_before_any_launch(what):
    alg, env = tracked_alg(), FakeEnv()
    ev_env = FakeEvalEnv(sync_stats=what == "sync_stats", num_obs=859 if what == "mismatch" else 860)
    kw = dict(eval_env=env if what == "same_core" else ev_env, eval_interval=2, eval_steps=4, eval_track_episodes=5)
    kw.update({"steps_odd": dict(eval_steps=3), "steps_zero": dict(eval_steps=0), "steps_none": dict(eval_steps=None),
               "interval_zero": dict(eval_interval=0), "interval_none": dict(eval_interval=None), "track_zero": dict(eval_track_episodes=0),
               "mode_unknown": dict(eval_modes=("teacher", "expert")), "modes_empty": dict(eval_modes=()),
               "modes_str": dict(eval_modes="student")}.get(what, {}))
    n0 = launches()
    with pytest.raises(L.DwbcError):
        GraphRunner(alg, env, **kw)
    assert launches() == n0 and ev_env.events == []


def test_learn_refuses_an_eval_core_changed_to_sync_stats():
    r, _, ev_env = make()
    ev_env.sync_stats = True
    with pytest.raises(L.DwbcError, match="sync_stats"):
        r.learn(1)
    assert r.current_learning_iteration == 0


@pytest.mark.parametrize("modes", [("teacher",), ("student",), ("student", "teacher")])
def test_evaluated_iterations_and_order(modes, tmp_path):
    r, env, ev_env = make(modes, interval=3, save_path=lambda it: str(tmp_path / f"model_{it}.pt"))
    events = []
    stub_launches(r, events)
    stub_evals(r, events)
    ev_env.events = events
    r.learn(4)
    r.learn(5)                                                     # continues at iteration 4
    order = [m for m in EVAL_MODES if m in modes]                  # the teacher first, whatever order the modes are given in
    want = []
    for it in range(9):
        dagger = it % 3 == 0
        want += [("rollout", dagger), "compute_returns", ("update_dagger", False) if dagger else ("update", False)]
        want += [] if dagger else ["enforce_min_std"]
        if it % 3 == 0:
            for m in order:
                want += ["restore", ("eval", m)]
    assert events == want
    rows = r.logs()
    assert [row["eval"] is not None for row in rows] == [it % 3 == 0 for it in range(9)]
    assert all(list(row["eval"]) == order for row in rows if row["eval"] is not None)
    assert not any(k in row for row in rows for k in TIMING_KEYS)

    r2, _, ev2 = make(modes, interval=3)                           # a resumed run at iteration 9 evaluates 9 and 12
    r2.load(str(tmp_path / "model_9.pt"))
    events.clear()
    stub_launches(r2, events)
    stub_evals(r2, events)
    r2.learn(4)
    rows = r2.logs()[9:]                                           # after the 9 rows the checkpoint carried unread
    assert [(row["iteration"], row["eval"] is not None) for row in rows] == [(9, True), (10, False), (11, False), (12, True)]
    assert [e for e in events if e[0] == "eval"] == [("eval", m) for m in order] * 2


def test_eval_rows_equal_the_readers_they_restate():
    """Hand-made trackers and statistics blocks for five evaluations: an empty ring, a partly filled one, one that wrapped more than
    twice, runs with and without ended episodes.  Each mode's entry equals statistics.mean over rsl_rl's deques (maxlen C), the
    tracker's count, and episode_stats() of a second env fed the same statistics in the same order (carrying over when none ended)."""
    cap = 5
    r, env, ev_env = make(cap=cap)
    ref = FakeEnv()
    g = torch.Generator().manual_seed(4)
    episodes = [tuple(float(x) for x in torch.randn(3, generator=g)) for _ in range(3 * cap + 2)]
    # per evaluation and mode: episodes appended in the run, episodes ended by the statistics
    plan = [((0, 0.0), (2, 2.0)), ((2, 3.0), (0, 0.0)), ((cap + 1, 2.0), (3 * cap + 2, 5.0)), ((3 * cap + 2, 0.0), (1, 1.0)),
            ((cap, 4.0), (cap - 1, 0.0))]
    state = {}

    def on_run(m):
        n_app, ended = state[m]
        ev = r._evals[m]
        assert not any(v.any() for v in ev._episodes.values())    # zeroed before the run
        fill_ring(ev, episodes[:n_app])
        ev_env._stats.copy_(torch.rand(ev_env._stats.numel(), generator=g) + 0.5)
        ev_env._stats[0] = ended
        state[m + ".stats"] = ev_env._stats.clone()
    stub_evals(r, [], on_run)
    want = []
    for it, per_mode in enumerate(plan):
        env.update_command_curriculum()
        for m, v in zip(EVAL_MODES, per_mode):
            state[m] = v
        r._snapshot(it, None)
        r._evaluate()
        row = {}
        for m, (n_app, _) in zip(EVAL_MODES, per_mode):
            means = deque_means(episodes[:n_app], cap)
            ref._stats.copy_(state[m + ".stats"])
            row[m] = dict(mean_reward=means[0], mean_arm_reward=means[1], mean_episode_length=means[2], num_episodes=n_app,
                          episode=dict(ref.episode_stats()))
        want.append(row)
    got = [row["eval"] for row in r.logs()]
    assert got == want
    assert got[3]["teacher"]["mean_reward"] is not None and got[0]["teacher"]["mean_reward"] is None
    key = "rew_" + ev_env.sum_names[0]
    assert torch.equal(got[1]["student"]["episode"][key], got[1]["teacher"]["episode"][key])   # none ended: carried over
    # the training curriculum moved, the evaluation task did not
    assert env.curriculum.update_counter == 5 and ev_env.curriculum.update_counter == 0
    assert got[0]["teacher"]["episode"]["coeff_lin_vel_x_upper_bound"] == got[4]["student"]["episode"]["coeff_lin_vel_x_upper_bound"]


class Clock:
    """Host stand-ins for torch.cuda.Event: record() takes the time of a clock the stubs advance (ms)."""
    now = 0

    def __init__(self, enable_timing=False):
        assert enable_timing
        self.t = None

    def record(self):
        self.t = Clock.now

    def elapsed_time(self, end):
        return end.t - self.t


def test_timing_fields_follow_from_the_event_times(monkeypatch):
    monkeypatch.setattr(GraphRunner, "_Event", Clock)
    Clock.now = 0
    r, env, ev_env = make(interval=2, log_interval=3, timing=True)
    events = []
    stub_launches(r, events)
    rollout, update = r.rollout.run, r.alg._ppo_run
    costs = dict(rollout=30, update=9, returns=1, eval=5)

    def tick(f, ms):
        def g(*a):
            Clock.now += ms
            return f(*a)
        return g
    r.rollout.run = tick(rollout, costs["rollout"])
    r.alg._ppo_run = tick(update, costs["update"])
    r.alg._dagger_run = tick(r.alg._dagger_run, 2 * costs["update"])
    r.alg.compute_returns = tick(r.alg.compute_returns, costs["returns"])
    stub_evals(r, events, on_run=lambda m: setattr(Clock, "now", Clock.now + costs["eval"]))
    r.alg.learning_rate = 3e-4
    r.learn(5)
    rows = r.logs()
    tot_steps, tot_time = 0, 0.0
    for it, row in enumerate(rows):
        collection = costs["rollout"] / 1e3
        learn = (costs["returns"] + (2 if it % 3 == 0 else 1) * costs["update"]) / 1e3
        tot_steps += T * N
        tot_time += collection + learn
        assert row["collection_time"] == collection and row["learn_time"] == learn
        assert row["fps"] == int(T * N / (collection + learn)) and row["tot_timesteps"] == tot_steps and row["tot_time"] == tot_time
        assert row["learning_rate"] == 3e-4 and row["captured"] is False
        assert ("eval_time" in row) == (it % 2 == 0)
        if it % 2 == 0:
            assert row["eval_time"] == 2 * costs["eval"] / 1e3
    assert r.tot_timesteps == 5 * T * N


def test_checkpoint_with_and_without_evaluation(tmp_path):
    alg, env = tracked_alg(dagger_update_freq=3), FakeEnv()
    plain = GraphRunner(alg, env, save_path=lambda it: str(tmp_path / f"plain_{it}.pt"))
    stub_launches(plain, env.events)
    plain.learn(1)
    assert set(torch.load(tmp_path / "plain_1.pt", weights_only=True)["dwbc"]) == {"alg", "env", "iteration", "logs", "episode"}
    assert "eval" not in plain.logs()[0]

    ev_env = FakeEvalEnv()
    ev_env._stats.fill_(0.25)
    ev_env.curriculum.update_counter = 4                           # the caller's evaluation task, taken at construction
    r, env, _ = make(interval=1, ev_env=ev_env, save_path=lambda it: str(tmp_path / f"eval_{it}.pt"))
    stub_launches(r, [])
    stub_evals(r, [])
    r.learn(2)
    ck = torch.load(tmp_path / "eval_2.pt", weights_only=True)
    assert set(ck["dwbc"]) == {"alg", "env", "iteration", "logs", "episode", "eval"}
    assert set(ck["dwbc"]["eval"]) == {"start", "episode"} and ck["dwbc"]["eval"]["start"]["update_counter"] == 4
    assert [row["eval"] is not None for row in ck["dwbc"]["logs"]] == [True, True]

    r2, _, ev2 = make(interval=1)
    r2.alg.counter = 40
    r2.load(str(tmp_path / "eval_2.pt"))
    assert r2.current_learning_iteration == 2 and r2.alg.counter == 2
    assert torch.equal(r2._eval_start["stats"], torch.full_like(ev2._stats, 0.25)) and r2._eval_start["update_counter"] == 4

    for runner, path in ((make(interval=1)[0], "plain_1.pt"), (GraphRunner(tracked_alg(), FakeEnv()), "eval_2.pt")):
        runner.alg.counter = 40
        with pytest.raises(L.DwbcError, match="evaluation snapshot"):
            runner.load(str(tmp_path / path))
        assert runner.alg.counter == 40 and runner.current_learning_iteration == 0    # nothing copied
