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

    python tools/runner_timing.py [--block 20] [--reps 7] [--warmup 1] [--out DIR]
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
    args = ap.parse_args()
    assert torch.cuda.is_available(), "runner_timing.py measures on a CUDA device"
    from graph_timing import gpu_info
    info = gpu_info()
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
