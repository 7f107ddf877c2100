"""GPU: GraphRunner computes what OnPolicyRunner.learn computes, bit for bit, and waits for the GPU only where it reads.

The reference is OPR.learn restated as an eager loop through the public API: per step act / env.step / process_env_step, then
compute_returns, update() or update_dagger() on the iterations `it % dagger_update_freq == 0` (OPR:129, 166-169), and every iteration
episode_buffers() with statistics.mean (OPR.log), env.episode_stats() and, with diagnostics, update_diagnostics().  On the workload of
tests/test_gpu_resume.py (the curriculum and the mixing / priv-reg / torque-supervision schedules moving at every iteration, a push step
in the first rollout, episodes ending) with dagger_update_freq = 3, GraphRunner eager (capture=False) and captured must leave every
parameter, Adam moment and step, `counter`, storage row, env-core tensor and tracker equal to the loop's (torch.equal), and log the same
values (compared as float64 bit patterns).  Further:
  * inside learn() nothing reads the device or synchronises (counted, and under torch.cuda.set_sync_debug_mode("error")); logs()
    then synchronises once;
  * log_interval 1, 3 and 7 give the same bits and rows;
  * 3 iterations, a checkpoint through save_path, fresh objects from other seeds, GraphRunner.load and 3 more iterations equal 6
    iterations straight, eager and graphs on either side of the save; the checkpoint's model_state_dict loads strictly into a
    FusedActorCritic;
  * each rollout key and each update kind is captured once over a run."""
import struct
import statistics

import numpy as np
import pytest
import torch

import test_gpu_resume as R
from test_gpu_cuda_graphs import _tensors, assert_bitwise

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
FREQ = 3                  # iterations 0, 3 and 6 of seven are student (DAgger) iterations
CAP = 100                 # the runner's deques (OPR: maxlen 100)


def build(monkeypatch, precision="tf32x3", H=10, N=4096, ts=False, seed=0, diagnostics=False):
    """tests/test_gpu_resume.py's workload with FusedPPO(track_episodes=CAP, diagnostics=...) and dagger_update_freq = FREQ."""
    from dwbc_b200 import ppo

    class Tracking(ppo.FusedPPO):
        def __init__(self, *a, **k):
            super().__init__(*a, track_episodes=CAP, diagnostics=diagnostics, **k)
    with monkeypatch.context() as m:
        m.setattr(ppo, "FusedPPO", Tracking)
        w = R.build(H, N, "flat", precision, ts, seed)
    w.alg.dagger_update_freq = FREQ
    return w


def opr_learn(w, iterations, init_at_random_ep_len=True):
    """OPR.learn (OPR:100-177) through the public API, reading every iteration; returns the rows OPR.log would see."""
    from dwbc_b200.runner import DAGGER_KEY, EPISODE_MEANS, PPO_KEYS
    env, alg, s = w.env, w.alg, w.alg.storage
    torch.cuda.manual_seed(11)
    if init_at_random_ep_len:
        env.episode_length_buf = torch.randint_like(env.episode_length_buf, high=int(env.max_episode_length))
    obs, rows = env.get_observations(), []
    for it in range(iterations):
        env.update_command_curriculum()
        hist_encoding = it % alg.dagger_update_freq == 0
        for t in range(R.T):
            actions = alg.act(obs, obs, hist_encoding)
            env.set_obs_target(s.obs_row(t + 1))
            env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
            obs, _, rewards, arm_rewards, dones, infos = env.step(actions, physics=lambda e, t=t: e.bind_sim(**w.pool[t]))
            alg.process_env_step(rewards, arm_rewards, dones, infos)
        alg.compute_returns(obs)
        row = dict(iteration=it, hist_encoding=hist_encoding)
        if hist_encoding:
            row[DAGGER_KEY] = alg.update_dagger()
        else:
            row.update(zip(PPO_KEYS, alg.update()))
        bufs = alg.episode_buffers()
        for buf, key in EPISODE_MEANS:
            row[key] = statistics.mean(bufs[buf]) if bufs[buf] else None
        row["episode"] = dict(env.episode_stats())
        row["std"] = alg.actor_critic.std.reshape(-1).tolist()
        if alg.diagnostics:
            row["diagnostics"] = None if hist_encoding else alg.update_diagnostics()
        rows.append(row)
    return rows


def runner(w, capture, log_interval=7, **kw):
    from dwbc_b200.runner import GraphRunner
    return GraphRunner(w.alg, w.env, physics=lambda t: w.env.bind_sim(**w.pool[t]), log_interval=log_interval, capture=capture, **kw)


def run_learn(r, iterations, init_at_random_ep_len=True):
    torch.cuda.manual_seed(11)
    r.learn(iterations, init_at_random_ep_len=init_at_random_ep_len)


def state(w):
    alg, env = w.alg, w.env
    out = dict(host=torch.tensor([env.common_step_counter, env.seed, env.curriculum.update_counter, alg.counter, alg.optimizer.step,
                                  alg.hist_encoder_optimizer.step]), generator=alg.generator.get_state())
    for prefix, obj in (("alg", alg), ("storage", alg.storage), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                        ("ac", alg.actor_critic), ("env", env)):
        out.update(_tensors(prefix, obj, skip=R.SKIP))
    out.update({f"tracker.{k}": v.clone() for k, v in alg._episodes.items()})
    out.update({f"sim.{k}": v.clone() for k, v in w.sim.items()})
    return out


def canon(x):
    """A logged value with every number as its float64 bit pattern (tensors, numpy and Python floats alike; NaN compares equal)."""
    if isinstance(x, dict):
        return {k: canon(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [canon(v) for v in x]
    if isinstance(x, (torch.Tensor, np.floating, float)) and not isinstance(x, bool):
        return struct.pack("<d", float(x)).hex()
    return x


def assert_rows(got, want):
    assert [r["iteration"] for r in got] == [r["iteration"] for r in want]
    for g, w_ in zip(got, want):
        assert canon(g) == canon(w_), g["iteration"]


def check_schedule(rows, iterations=7):
    assert [r["hist_encoding"] for r in rows] == [it % FREQ == 0 for it in range(iterations)]
    assert rows[-1]["mean_reward"] is not None and rows[-1]["episode"]            # episodes ended
    mix = [r["mean_value_mixing_ratio"] for r in rows if not r["hist_encoding"]]
    assert len(set(mix)) > 1                                                        # the schedules moved


class Captures:
    """How often RolloutGraph and FusedPPO capture, by rollout key flag / update kind."""

    def __init__(self, monkeypatch):
        from dwbc_b200.graphs import RolloutGraph
        from dwbc_b200.ppo import FusedPPO
        self.seen = []
        for cls, which in ((RolloutGraph, lambda a: ("rollout", a[1])), (FusedPPO, lambda a: ("update", a[0]))):
            orig = cls._capture
            monkeypatch.setattr(cls, "_capture", lambda self_, *a, _o=orig, _w=which: (self.seen.append(_w(a)), _o(self_, *a))[1])


# precision, history_len, envs, torque supervision: the TMA post-physics kernel at 4096 envs, the warp-per-env kernel at 1000 envs
CASES = [("fp32", 10, 4096, False), ("tf32x3", 10, 4096, False), ("tf32x3", 10, 4096, True), ("fp32", 20, 1000, False),
         ("tf32x3", 20, 1000, False)]
IDS = ["fp32-4096", "tf32x3-4096", "tf32x3-4096-ts", "fp32-h20-1000", "tf32x3-h20-1000"]


@pytest.mark.parametrize("precision,H,N,ts", CASES, ids=IDS)
def test_runner_equals_opr_learn_restated(precision, H, N, ts, monkeypatch):
    w = build(monkeypatch, precision, H, N, ts)
    want_rows = opr_learn(w, 7)
    want, want_entropy = state(w), w.alg.last_entropy
    R.free(w)
    check_schedule(want_rows)
    assert ts == any(r["mean_arm_torques_loss"] != 0.0 for r in want_rows if not r["hist_encoding"])
    for capture in (False, True):
        w = build(monkeypatch, precision, H, N, ts)
        cap = Captures(monkeypatch)
        r = runner(w, capture)
        run_learn(r, 7)
        rows = r.logs()
        assert_bitwise(want, state(w))
        assert_rows(rows, want_rows)
        assert w.alg.last_entropy == want_entropy
        if capture:                                   # each rollout key and each update kind captured once over the run
            assert sorted(cap.seen) == [("rollout", False), ("rollout", True), ("update", "dagger"), ("update", "ppo")], cap.seen
        else:
            assert cap.seen == []
        monkeypatch.undo()
        del r
        R.free(w)


class Waits:
    """Counts the calls that wait for the device: synchronize of the device, a stream or an event, and item / tolist / cpu of a CUDA
    tensor."""

    def __init__(self, monkeypatch):
        self.calls = []

        def wrap(owner, name, cuda_only=False):
            orig = getattr(owner, name)

            def counted(*a, **k):
                if not cuda_only or (isinstance(a[0], torch.Tensor) and a[0].is_cuda):
                    self.calls.append(f"{getattr(owner, '__name__', owner)}.{name}")
                return orig(*a, **k)
            monkeypatch.setattr(owner, name, counted)
        wrap(torch.cuda, "synchronize")
        wrap(torch.cuda.Stream, "synchronize")
        wrap(torch.cuda.Event, "synchronize")
        for name in ("item", "tolist", "cpu"):
            wrap(torch.Tensor, name, cuda_only=True)


@pytest.mark.parametrize("capture", [False, True], ids=["eager", "graphs"])
def test_learn_does_not_wait_for_the_gpu(capture, monkeypatch):
    w = build(monkeypatch)
    r = runner(w, capture, log_interval=7)
    run_learn(r, 2)                                   # iterations 0 (DAgger) and 1 (PPO): every graph is captured here
    r.logs()
    waits = Waits(monkeypatch)
    torch.cuda.set_sync_debug_mode("error")
    try:
        r.learn(7)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert waits.calls == [], waits.calls
    rows = r.logs()
    assert waits.calls == ["Stream.synchronize"], waits.calls
    assert [row["iteration"] for row in rows] == list(range(2, 9))
    monkeypatch.undo()
    del r
    R.free(w)


def test_log_interval_does_not_change_bits_or_rows(monkeypatch):
    out = {}
    for interval in (1, 3, 7):
        w = build(monkeypatch)
        r = runner(w, True, log_interval=interval)
        run_learn(r, 7)
        out[interval] = (state(w), r.logs())
        del r
        R.free(w)
    check_schedule(out[7][1])
    for interval in (1, 3):
        assert_bitwise(out[7][0], out[interval][0])
        assert_rows(out[interval][1], out[7][1])


@pytest.mark.parametrize("capture_before,capture_after", [(False, True), (True, False), (True, True)],
                         ids=["eager-graphs", "graphs-eager", "graphs-graphs"])
def test_resumed_learn_equals_straight_learn(capture_before, capture_after, monkeypatch, tmp_path):
    from dwbc_b200.runner_compat import FusedActorCritic
    w = build(monkeypatch)
    r = runner(w, capture_before)
    run_learn(r, 6)
    straight, straight_rows = state(w), r.logs()
    del r
    R.free(w)

    w = build(monkeypatch)
    saved = []
    r = runner(w, capture_before, log_interval=2, save_path=lambda it: (saved.append(it), str(tmp_path / f"model_{it}.pt"))[1])
    run_learn(r, 3)
    sim = {k: v.clone() for k, v in w.sim.items()}              # the simulator's state is the caller's to keep
    del r
    R.free(w)
    assert saved == [0, 3]                                       # it % save_interval == 0 (OPR:175-176), and after the last iteration

    ck = torch.load(tmp_path / "model_3.pt", weights_only=True)
    assert set(ck) == {"model_state_dict", "optimizer_state_dict", "iter", "infos", "dwbc"} and ck["iter"] == 3
    policy = FusedActorCritic(76, 76, 18, actor_hidden_dims=(128,), critic_hidden_dims=(128,), num_priv=24, num_hist=10, num_prop=76,
                              device=DEV)
    policy.load_state_dict(ck["model_state_dict"])               # strict: the reference's key names and shapes
    assert all(torch.equal(v, ck["model_state_dict"][k]) for k, v in policy.state_dict().items())

    w = build(monkeypatch, seed=1)
    assert w.alg.counter == 0 and w.env.curriculum.update_counter == 3
    for k, v in w.sim.items():
        v.copy_(sim[k])
    r = runner(w, capture_after)
    r.load(str(tmp_path / "model_3.pt"))
    assert r.current_learning_iteration == 3
    r.learn(3)
    resumed, resumed_rows = state(w), r.logs()
    del r
    R.free(w)
    assert [row["hist_encoding"] for row in straight_rows] == [True, False, False, True, False, False]   # a DAgger iteration after the save
    assert_rows(resumed_rows, straight_rows)
    assert_bitwise(straight, resumed)


@pytest.mark.parametrize("capture", [False, True], ids=["eager", "graphs"])
def test_logged_diagnostics_equal_update_diagnostics(capture, monkeypatch):
    w = build(monkeypatch, diagnostics=True)
    want_rows = opr_learn(w, 7)
    want = state(w)
    R.free(w)
    w = build(monkeypatch, diagnostics=True)
    r = runner(w, capture)
    run_learn(r, 7)
    rows = r.logs()
    assert [row["diagnostics"] is None for row in rows] == [it % FREQ == 0 for it in range(7)]
    assert all(row["diagnostics"]["per_minibatch"]["grad_norm"] for row in rows if row["diagnostics"] is not None)
    assert_rows(rows, want_rows)
    assert_bitwise(want, state(w))
    del r
    R.free(w)
