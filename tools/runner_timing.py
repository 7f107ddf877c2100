#!/usr/bin/env python
"""What reading results once per log interval instead of once per iteration saves, on bench.py's flat workload (4096 envs, T = 40,
tf32x3, 5 epochs x 4 mini-batches, dagger_update_freq 20, FusedPPO(track_episodes=100)).

Three arms, each on its own objects built from the same seeds, all captured (RolloutGraph, FusedPPO(cuda_graphs=True)):
  (a) INTEGRATION §3.3's hand-written loop with OPR.learn's teacher / student alternation: update() / update_dagger(), then
      env.episode_stats() and alg.episode_buffers() with statistics.mean, so the host waits for the GPU at least once per iteration;
  (b) GraphRunner(capture=True, log_interval=1), logs() after every iteration;
  (c) GraphRunner(capture=True, log_interval=20), logs() after every block.
The arms run in turn, one block of --block iterations each, --reps times after --warmup blocks.  Per block: the wall time from the
first enqueue to the end of a device synchronise (iteration time = block time / block), the host wall time until the loop returns
(before the final synchronise; for (a) it includes its per-iteration waits) and the process CPU time (which includes the host spinning
in a synchronise).  A separate phase then profiles one block of each arm with torch.profiler and reports the GPU idle time: the span
from the first to the last GPU activity minus the union of the kernel / memcpy / memset intervals, per iteration, and the largest gap.
All arms must end with bitwise-equal parameters.  The card's name, power limit and clocks are read in the same run.

With --eval-interval, the cost of scheduled evaluation and of the timing events instead: two arms of GraphRunner(capture=True,
log_interval=--block) on the same workload, both evaluating the teacher and the student (--eval-steps steps) every --eval-interval
iterations on a second core (bench.py's workload of rank 1), one with timing=True's events and one without, alternating blocks as above.
Reported: the iteration time of each arm, the rows' GPU times (collection, learning, evaluation per evaluated iteration), the GPU time
of one mode's evaluation alone (CUDA events around the snapshot restore and the EvalGraph replay, per mode), and the host time that
enqueueing an evaluation adds to an evaluated iteration.  Both arms must end with bitwise-equal parameters.

    python tools/runner_timing.py [--block 20] [--reps 7] [--warmup 1] [--out DIR]
    python tools/runner_timing.py --eval-interval 10 --eval-steps 1000 [--block 20] [--reps 7] [--warmup 1] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

ARMS = ("a_loop", "b_runner_1", "c_runner_20")


def build(arm):
    import bench
    from dwbc_b200 import ppo
    from dwbc_b200.graphs import RolloutGraph
    from dwbc_b200.runner import GraphRunner
    orig = ppo.FusedPPO

    class Tracking(orig):
        def __init__(self, *a, **k):
            super().__init__(*a, track_episodes=100, cuda_graphs=True, **k)
    ppo.FusedPPO = Tracking
    try:
        w = bench.Workload("cuda:0", 0, precision="tf32x3")
    finally:
        ppo.FusedPPO = orig
    physics = lambda t: w.env.bind_sim(**w.pool[t])  # noqa: E731
    if arm == "a_loop":
        w.rg, w.it = RolloutGraph(w.alg, w.env, physics), 0
    else:
        w.runner = GraphRunner(w.alg, w.env, physics, log_interval=1 if arm == "b_runner_1" else 20, capture=True)
    return w


def block(arm, w, n):
    """n iterations of the arm; returns the rows it logged."""
    if arm != "a_loop":
        r = w.runner
        if arm == "b_runner_1":
            rows = []
            for _ in range(n):
                r.learn(1)
                rows += r.logs()
            return rows
        r.learn(n)
        return r.logs()
    env, alg, rows = w.env, w.alg, []
    obs = env.get_observations()
    for it in range(w.it, w.it + n):
        env.update_command_curriculum()
        hist_encoding = it % alg.dagger_update_freq == 0
        obs = w.rg.run(obs, hist_encoding)
        alg.compute_returns(obs)
        losses = alg.update_dagger() if hist_encoding else alg.update()
        episode = env.episode_stats()
        bufs = alg.episode_buffers()
        rows.append(dict(losses=losses, episode=episode, mean_reward=statistics.mean(bufs["rewbuffer"]) if bufs["rewbuffer"] else None,
                         mean_episode_length=statistics.mean(bufs["lenbuffer"]) if bufs["lenbuffer"] else None))
    w.it += n
    return rows


def build_eval(timing, args):
    """bench.py's workload under a GraphRunner that evaluates on the core of a second workload (rank 1)."""
    import bench
    from dwbc_b200 import ppo
    from dwbc_b200.runner import GraphRunner
    orig = ppo.FusedPPO

    class Tracking(orig):
        def __init__(self, *a, **k):
            super().__init__(*a, track_episodes=100, **k)
    ppo.FusedPPO = Tracking
    try:
        w = bench.Workload("cuda:0", 0, precision="tf32x3")
        ev = bench.Workload("cuda:0", 1, precision="tf32x3")
    finally:
        ppo.FusedPPO = orig
    w.ev = ev
    w.runner = GraphRunner(w.alg, w.env, lambda t: w.env.bind_sim(**w.pool[t]), log_interval=args.block, capture=True, eval_env=ev.env,
                           eval_interval=args.eval_interval, eval_steps=args.eval_steps,
                           eval_physics=lambda t: ev.env.bind_sim(**ev.pool[t % len(ev.pool)]), timing=timing)
    w.enqueue = []                                      # host seconds spent enqueueing each evaluation
    evaluate = w.runner._evaluate

    def timed():
        t0 = time.perf_counter()
        evaluate()
        w.enqueue.append(time.perf_counter() - t0)
    w.runner._evaluate = timed
    return w


def eval_main(args, info):
    arms = ("timing_off", "timing_on")
    work = {arm: build_eval(arm == "timing_on", args) for arm in arms}
    for _ in range(args.warmup):
        for arm in arms:
            work[arm].runner.learn(args.block)
            work[arm].runner.logs()
    res, rows = {arm: [] for arm in arms}, []
    for arm in arms:
        work[arm].enqueue.clear()
    for _ in range(args.reps):
        for arm in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            work[arm].runner.learn(args.block)
            torch.cuda.synchronize()
            res[arm].append(1e3 * (time.perf_counter() - t0) / args.block)
            out = work[arm].runner.logs()
            if arm == "timing_on":
                rows += out
    med = lambda v: dict(median=statistics.median(v), min=min(v), max=max(v), n=len(v))  # noqa: E731
    r = work["timing_on"].runner
    per_mode = {}
    for m, g in r._evals.items():                       # one mode alone: restore + replay, between CUDA events
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r.eval_env.load_state_dict(r._eval_start)
            for v in g._episodes.values():
                v.zero_()
            g.run(r.eval_env.obs_buf)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        per_mode[m] = med(times)
    evaluated = [row for row in rows if "eval_time" in row]
    out = dict(gpu=info, block=args.block, reps=args.reps, warmup=args.warmup, eval_interval=args.eval_interval, eval_steps=args.eval_steps,
               iteration_ms={arm: med(v) for arm, v in res.items()},
               rows=dict(collection_ms=med([1e3 * x["collection_time"] for x in rows]), learn_ms=med([1e3 * x["learn_time"] for x in rows]),
                         fps=med([x["fps"] for x in rows]), eval_ms=med([1e3 * x["eval_time"] for x in evaluated]),
                         captured_rows=sum(x["captured"] for x in rows)),
               eval_mode_ms=per_mode, eval_enqueue_host_ms={arm: med([1e3 * t for t in work[arm].enqueue]) for arm in arms},
               last_eval={m: {k: v for k, v in e.items() if k != "episode"} for m, e in evaluated[-1]["eval"].items()},
               parameters_equal=bool(torch.equal(work["timing_off"].alg.actor_critic.flat, work["timing_on"].alg.actor_critic.flat)))
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "runner_eval_timing.json"), "w") as f:
            json.dump(out, f, indent=1)
    assert out["parameters_equal"]


def gpu_idle(prof, n):
    """GPU idle time (ms per iteration) over the profiled block and the largest single gap (ms)."""
    spans = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start)
    busy, gap_max, cur_s, cur_e = 0.0, 0.0, None, None
    for s, e in spans:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                busy += cur_e - cur_s
                gap_max = max(gap_max, s - cur_e)
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = spans[-1][1] - spans[0][0]
    return dict(idle_ms_per_iteration=(span - busy) / 1e3 / n, largest_gap_ms=gap_max / 1e3, gpu_span_ms_per_iteration=span / 1e3 / n,
                activities=len(spans))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block", type=int, default=20, help="iterations per timed block (c's log interval is 20)")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--eval-interval", type=int, default=None, help="measure scheduled evaluation every this many iterations instead")
    ap.add_argument("--eval-steps", type=int, default=1000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "runner_timing.py measures on a CUDA device"
    from graph_timing import gpu_info
    info = gpu_info()
    if args.eval_interval is not None:
        return eval_main(args, info)
    work = {arm: build(arm) for arm in ARMS}
    for _ in range(args.warmup):
        for arm in ARMS:
            block(arm, work[arm], args.block)
    torch.cuda.synchronize()
    res = {arm: dict(iteration_ms=[], host_ms=[], cpu_ms=[]) for arm in ARMS}
    last_rows = {}
    for _ in range(args.reps):
        for arm in ARMS:
            torch.cuda.synchronize()
            t0, c0 = time.perf_counter(), time.process_time()
            last_rows[arm] = block(arm, work[arm], args.block)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            t2, c2 = time.perf_counter(), time.process_time()
            res[arm]["iteration_ms"].append(1e3 * (t2 - t0) / args.block)
            res[arm]["host_ms"].append(1e3 * (t1 - t0) / args.block)
            res[arm]["cpu_ms"].append(1e3 * (c2 - c0) / args.block)
    summary = {arm: {k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in r.items()} for arm, r in res.items()}
    from torch.profiler import ProfilerActivity, profile
    for arm in ARMS:                                    # separate phase: tracing slows the host
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            block(arm, work[arm], args.block)
            torch.cuda.synchronize()
        summary[arm]["profiled"] = gpu_idle(prof, args.block)
    flats = {arm: work[arm].alg.actor_critic.flat for arm in ARMS}
    equal = {arm: bool(torch.equal(flats["a_loop"], flats[arm])) for arm in ARMS}
    rewards = {arm: [r["mean_reward"] for r in last_rows[arm]][-1] for arm in ARMS}
    out = dict(gpu=info, block=args.block, reps=args.reps, warmup=args.warmup, parameters_equal_to_a=equal, last_mean_reward=rewards,
               iterations_per_arm=args.block * (args.warmup + args.reps + 1), arms=summary)
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "runner_timing.json"), "w") as f:
            json.dump(out, f, indent=1)
    assert all(equal.values()), equal


if __name__ == "__main__":
    main()
