"""GPU: GraphRunner's scheduled evaluation logs what OPR.learn with evaluations between its iterations logs, bit for bit, without
waiting for the GPU, and training does not see it.

The reference is tests/test_gpu_graph_runner.py's OPR.learn restated as an eager loop, with an evaluation after the update of every
iteration `it % EVAL_INTERVAL == 0` through public calls: per mode (teacher, then student), `eval_env.load_state_dict(snapshot)` of the
state_dict() taken before training, a fresh `EvalGraph(capture=False).run`, `results()` with statistics.mean.  The evaluation core is a
second core whose simulator stand-in copies fixed per-step tensors into the buffers it binds, so a run's inputs do not depend on earlier
runs.  Further:
  * training with and without evaluation leaves every training tensor and row equal, and timing=False records no event;
  * two evaluations of unchanged parameters (learning rate 0) log the same values; every mode's run starts from the same core tensors;
  * learn() with evaluation and timing makes no synchronising call, logs() one; every eval mode is captured once per run;
  * 3 iterations, a checkpoint, fresh objects from other seeds (the eval core too), load and 3 more equal 6 straight iterations;
    log_interval 1, 3 and 7 give the same rows;
  * timing fields are finite, positive and consistent, with eval_time on evaluated iterations only."""
import math
import statistics

import pytest
import torch

import test_gpu_eval_graph as EG
import test_gpu_graph_runner as GR
import test_gpu_resume as R
from test_gpu_cuda_graphs import _tensors, assert_bitwise

pytestmark = pytest.mark.gpu

EVAL_INTERVAL, EVAL_STEPS, EVAL_CAP = 2, 40, 100
SIM = ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")


def eval_core(w, seed=0):
    """A second core of w's configuration with its own Philox seed and a start the caller sets (curriculum, random episode lengths, an
    observation); seed != 0 gives it another state, which a checkpoint's snapshot replaces.  physics(t) copies pool[t % 24] into fixed
    buffers and binds them."""
    env, pool, obs0 = EG.make_core(w.p.history_len, w.p.num_envs, "flat", seed=2000 + seed)
    for _ in range(2 + seed):
        env.update_command_curriculum()
    g = torch.Generator(device=GR.DEV)
    g.manual_seed(77 + seed)
    env.episode_length_buf = torch.randint(0, int(env.max_episode_length), env.episode_length_buf.shape, device=GR.DEV, generator=g)
    env.obs_buf[:, :env.num_obs].copy_(obs0 * (1 + seed))
    env.common_step_counter += 5 * seed
    work = {k: pool[0][k].clone() for k in SIM}

    def physics(t):
        for k in SIM:
            work[k].copy_(pool[t % len(pool)][k])
        env.bind_sim(**work)
    return env, physics


def runner(w, ev, capture, log_interval=7, modes=("teacher", "student"), **kw):
    from dwbc_b200.runner import GraphRunner
    return GraphRunner(w.alg, w.env, physics=lambda t: w.env.bind_sim(**w.pool[t]), log_interval=log_interval, capture=capture,
                       eval_env=ev[0], eval_physics=ev[1], eval_interval=EVAL_INTERVAL, eval_steps=EVAL_STEPS,
                       eval_track_episodes=EVAL_CAP, eval_modes=modes, **kw)


def evaluate(w, ev, snapshot):
    """One scheduled evaluation through public calls."""
    from dwbc_b200.graphs import EvalGraph
    from dwbc_b200.runner import EPISODE_MEANS
    env, physics = ev
    out = {}
    for mode in ("teacher", "student"):
        env.load_state_dict(snapshot)
        g = EvalGraph(w.alg.actor_critic, env, EVAL_STEPS, hist_encoding=mode == "student", track_episodes=EVAL_CAP, physics=physics,
                      capture=False)
        g.run(env.obs_buf)
        res = g.results()
        out[mode] = {key: statistics.mean(res[buf]) if res[buf] else None for buf, key in EPISODE_MEANS}
        out[mode].update(num_episodes=int(g._episodes["pos"][1]), episode=dict(res["episode"]))
    return out


def opr_learn_eval(w, ev, iterations):
    """GR.opr_learn with an evaluation after the update of every iteration it % EVAL_INTERVAL == 0."""
    snapshot, alg, evals = ev[0].state_dict(), w.alg, []
    for name in ("update", "update_dagger"):
        orig = getattr(alg, name)

        def hooked(*a, _orig=orig):
            out = _orig(*a)
            it = len(evals)
            evals.append(evaluate(w, ev, snapshot) if it % EVAL_INTERVAL == 0 else None)
            return out
        setattr(alg, name, hooked)
    rows = GR.opr_learn(w, iterations)
    del alg.update, alg.update_dagger
    for row, e in zip(rows, evals):
        row["eval"] = e
    return rows


def eval_state(ev, skip=()):
    return _tensors("eval", ev[0], skip=R.SKIP + ("_dev_step",) + skip)


class EvalCaptures(GR.Captures):
    def __init__(self, monkeypatch):
        super().__init__(monkeypatch)
        from dwbc_b200.graphs import EvalGraph
        orig = EvalGraph._capture
        monkeypatch.setattr(EvalGraph, "_capture", lambda g, *a: (self.seen.append(("eval", g.hist_encoding)), orig(g, *a))[1])


def check_evals(rows):
    assert [r["eval"] is not None for r in rows] == [r["iteration"] % EVAL_INTERVAL == 0 for r in rows]
    done = [r["eval"] for r in rows if r["eval"] is not None]
    assert all(e[m]["num_episodes"] > 0 and e[m]["mean_reward"] is not None for e in done for m in e)          # episodes ended
    assert GR.canon(done[0]["teacher"]) != GR.canon(done[-1]["teacher"]) != GR.canon(done[-1]["student"])


CASES = [("fp32", 10, 4096), ("tf32x3", 10, 4096), ("tf32x3", 20, 1000)]
IDS = ["fp32-4096", "tf32x3-4096", "tf32x3-h20-1000"]


@pytest.mark.parametrize("precision,H,N", CASES, ids=IDS)
def test_runner_evaluations_equal_the_restated_loop(precision, H, N, monkeypatch):
    w = GR.build(monkeypatch, precision, H, N)
    ev = eval_core(w)
    want_rows = opr_learn_eval(w, ev, 7)
    want, want_eval = GR.state(w), eval_state(ev)
    R.free(w)
    del ev
    check_evals(want_rows)
    for capture in (False, True):
        w = GR.build(monkeypatch, precision, H, N)
        ev = eval_core(w)
        cap = EvalCaptures(monkeypatch)
        r = runner(w, ev, capture)
        GR.run_learn(r, 7)
        rows = r.logs()
        GR.assert_rows(rows, want_rows)
        assert_bitwise(want, GR.state(w))
        assert_bitwise(want_eval, eval_state(ev))
        if capture:
            assert sorted(cap.seen) == [("eval", False), ("eval", True), ("rollout", False), ("rollout", True), ("update", "dagger"),
                                        ("update", "ppo")], cap.seen
        else:
            assert cap.seen == []
        monkeypatch.undo()
        del r, ev
        R.free(w)


def test_training_does_not_see_the_evaluations(monkeypatch):
    from dwbc_b200.runner import TIMING_KEYS
    w = GR.build(monkeypatch)
    r = GR.runner(w, True)
    GR.run_learn(r, 7)
    plain, plain_rows = GR.state(w), r.logs()
    del r
    R.free(w)
    records = []
    monkeypatch.setattr(torch.cuda.Event, "record", lambda *a, **k: records.append(a))
    w = GR.build(monkeypatch)
    r = runner(w, eval_core(w), True)
    GR.run_learn(r, 7)
    rows = r.logs()
    assert records == [] and r._events is None and not any(k in row for row in rows for k in TIMING_KEYS)
    check_evals(rows)
    assert_bitwise(plain, GR.state(w))
    GR.assert_rows([{k: v for k, v in row.items() if k != "eval"} for row in rows], plain_rows)
    del r
    R.free(w)


def test_evaluations_of_unchanged_parameters_repeat(monkeypatch):
    from dwbc_b200.graphs import EvalGraph
    w = GR.build(monkeypatch)
    w.alg.learning_rate = 0.0                              # the Adam steps move nothing: every evaluation sees the same parameters
    flat = w.alg.actor_critic.flat.clone()
    ev = eval_core(w)
    starts, orig = [], EvalGraph.run

    def run(g, obs):
        starts.append(dict(eval_state(ev, skip=R.SIM), obs=obs[:, :ev[0].num_obs].clone(), step=torch.tensor(ev[0].common_step_counter)))
        return orig(g, obs)
    monkeypatch.setattr(EvalGraph, "run", run)
    from dwbc_b200.runner import GraphRunner
    r = GraphRunner(w.alg, w.env, physics=lambda t: w.env.bind_sim(**w.pool[t]), log_interval=7, capture=True, eval_env=ev[0],
                    eval_physics=ev[1], eval_interval=1, eval_steps=EVAL_STEPS, eval_track_episodes=EVAL_CAP)
    GR.run_learn(r, 4)
    rows = r.logs()
    assert torch.equal(flat, w.alg.actor_critic.flat)
    assert len(starts) == 8
    for s in starts[1:]:
        assert_bitwise(starts[0], s)
    evals = [GR.canon(row["eval"]) for row in rows]
    assert all(e == evals[0] for e in evals) and evals[0]["teacher"] != evals[0]["student"]
    del r
    R.free(w)


@pytest.mark.parametrize("capture", [False, True], ids=["eager", "graphs"])
def test_learn_with_evaluation_and_timing_does_not_wait(capture, monkeypatch):
    from dwbc_b200.runner import TIMING_KEYS
    w = GR.build(monkeypatch)
    r = runner(w, eval_core(w), capture, timing=True)
    GR.run_learn(r, 2)                                     # iteration 0 (DAgger, evaluated) and 1 (PPO): every graph is captured here
    rows = r.logs()
    waits = GR.Waits(monkeypatch)
    torch.cuda.set_sync_debug_mode("error")
    try:
        r.learn(7)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert waits.calls == [], waits.calls
    rows += r.logs()
    assert waits.calls == ["Stream.synchronize"], waits.calls
    monkeypatch.undo()
    assert [row["iteration"] for row in rows] == list(range(9))
    check_evals(rows)
    steps, tot = w.alg.storage.num_transitions_per_env * w.alg.storage.num_envs, 0.0
    for i, row in enumerate(rows):
        assert set(TIMING_KEYS) - {"eval_time"} <= set(row) and ("eval_time" in row) == (row["iteration"] % EVAL_INTERVAL == 0)
        times = [row["collection_time"], row["learn_time"]] + ([row["eval_time"]] if "eval_time" in row else [])
        assert all(math.isfinite(t) and t > 0 for t in times), row
        tot += row["collection_time"] + row["learn_time"]
        assert row["fps"] == int(steps / (row["collection_time"] + row["learn_time"])) and row["fps"] > 0
        assert row["tot_timesteps"] == (i + 1) * steps and math.isclose(row["tot_time"], tot, rel_tol=1e-12)
        assert row["learning_rate"] == w.alg.learning_rate
        assert row["captured"] == (capture and i < 2)
    print("timing rows:", [(row["iteration"], round(1e3 * row["collection_time"], 2), round(1e3 * row["learn_time"], 2),
                            round(1e3 * row.get("eval_time", 0), 2), row["captured"]) for row in rows])
    del r
    R.free(w)


@pytest.mark.parametrize("capture_before,capture_after", [(False, True), (True, False), (True, True)],
                         ids=["eager-graphs", "graphs-eager", "graphs-graphs"])
def test_resumed_learn_with_evaluation_equals_straight_learn(capture_before, capture_after, monkeypatch, tmp_path):
    w = GR.build(monkeypatch)
    ev = eval_core(w)
    r = runner(w, ev, capture_before)
    GR.run_learn(r, 6)
    straight, straight_rows = GR.state(w), r.logs()
    del r, ev
    R.free(w)
    check_evals(straight_rows)

    w = GR.build(monkeypatch)
    r = runner(w, eval_core(w), capture_before, log_interval=2, save_path=lambda it: str(tmp_path / f"model_{it}.pt"))
    GR.run_learn(r, 3)
    sim = {k: v.clone() for k, v in w.sim.items()}
    del r
    R.free(w)
    ck = torch.load(tmp_path / "model_3.pt", weights_only=True)
    assert set(ck["dwbc"]["eval"]) == {"start", "episode"}

    w = GR.build(monkeypatch, seed=1)
    for k, v in w.sim.items():
        v.copy_(sim[k])
    other = eval_core(w, seed=1)
    before = other[0].state_dict()
    r = runner(w, other, capture_after)
    assert not torch.equal(r._eval_start["tensors"]["episode_length_buf"], ck["dwbc"]["eval"]["start"]["tensors"]["episode_length_buf"])
    r.load(str(tmp_path / "model_3.pt"))
    r.learn(3)
    resumed, resumed_rows = GR.state(w), r.logs()
    del r, other, before
    R.free(w)
    GR.assert_rows(resumed_rows, straight_rows)
    assert_bitwise(straight, resumed)


def test_log_interval_does_not_change_evaluations(monkeypatch):
    out = {}
    for interval in (1, 3, 7):
        w = GR.build(monkeypatch)
        r = runner(w, eval_core(w), True, log_interval=interval)
        GR.run_learn(r, 7)
        out[interval] = (GR.state(w), r.logs())
        del r
        R.free(w)
    check_evals(out[7][1])
    for interval in (1, 3):
        assert_bitwise(out[7][0], out[interval][0])
        GR.assert_rows(out[interval][1], out[7][1])
