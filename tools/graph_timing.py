#!/usr/bin/env python
"""Eager against CUDA-graph replay on bench.py's flat workload (T = 40, tf32x3, 5 epochs x 4 mini-batches) at --hist history steps and
--envs envs (default 10 and 4096: bench.py's own workload; built by tools/history_bench.py's workload()).

Two workloads from the same seeds, one eager and one with a captured rollout (dwbc_b200.graphs.RolloutGraph) and captured update()
(FusedPPO(cuda_graphs=True)), run one iteration each in turn, --runs times (after --warmup iterations each).  Per iteration it records
the rollout, update() and whole-iteration times (CUDA events), the host CPU time of the process (time.process_time; it includes the time
the host waits in the iteration's one synchronisation), the host wall time spent enqueueing the rollout, and the library calls made
through the ctypes binding.  Which post-physics kernel ran is read from derived_state column 27 (the TMA kernel's out-of-range history
counter; the warp-per-env kernel leaves it at 0).  The card's name, power limit and clocks are read in the same run.

With --track-episodes C two more arms run FusedPPO(track_episodes=C) (the runner's episode bookkeeping on the device, one
dwbc_track_episodes launch per env step), eagerly and captured, alternating with the two untracked arms.  The tracker's own time per
step is then measured with CUDA events around 1000 queued launches on synthetic inputs (2 % dones) at --envs and at 40 000 envs, issued
eagerly and replayed from a CUDA graph.

    python tools/graph_timing.py [--hist 10] [--envs 4096] [--runs 5] [--warmup 3] [--track-episodes C] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


class CountingLib:
    """The ctypes library with a call counter in front of every function."""

    def __init__(self, lib):
        self._lib, self.calls = lib, 0

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not callable(fn):
            return fn

        def call(*a):
            self.calls += 1
            return fn(*a)
        return call


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout
        return dict(zip(q.split(","), [x.strip() for x in out.strip().splitlines()[0].split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def tracker_step_us(L, n, cap, launches=1000):
    """Mean time of one dwbc_track_episodes launch at n envs (us): CUDA events around `launches` queued launches, issued eagerly (which
    the host's launch rate can bound) and replayed from a CUDA graph."""
    g = torch.Generator(device="cuda:0")
    g.manual_seed(3)
    rew, arm = (torch.randn(n, device="cuda:0", generator=g) for _ in range(2))
    dones = torch.rand(n, device="cuda:0", generator=g) < 0.02
    running, ring, pos = torch.zeros(n, 3, device="cuda:0"), torch.zeros(cap, 3, device="cuda:0"), torch.zeros(2, dtype=torch.int64, device="cuda:0")
    lib = L.lib()

    def launch():
        L.check(lib.dwbc_track_episodes(L.ptr(rew), L.ptr(arm), L.ptr(dones), n, L.ptr(running), L.ptr(ring), L.ptr(pos), cap,
                                        L.stream_ptr()), "dwbc_track_episodes")
    for _ in range(50):
        launch()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    for _ in range(launches):
        launch()
    ev[1].record()
    graph = torch.cuda.CUDAGraph()                      # the same launches replayed from a graph, as in a captured rollout
    with torch.cuda.graph(graph):
        for _ in range(launches):
            launch()
    graph.replay()
    ev[2].record()
    graph.replay()
    ev[3].record()
    torch.cuda.synchronize()
    return dict(eager=1e3 * ev[0].elapsed_time(ev[1]) / launches, graph=1e3 * ev[2].elapsed_time(ev[3]) / launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hist", type=int, default=10, choices=[10, 20, 50], help="history_len (StateHistoryEncoder tsteps)")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--track-episodes", type=int, default=0, help="C > 0: also run the arms with FusedPPO(track_episodes=C)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "graph_timing.py measures on a CUDA device"
    from history_bench import workload
    from dwbc_b200 import _lib as L
    from dwbc_b200.graphs import RolloutGraph
    counting = CountingLib(L.lib())
    L._lib = counting                                   # FusedPPO / the env core / the storage bind L.lib() at construction

    arms = {}
    for track in ((0, args.track_episodes) if args.track_episodes else (0,)):
        for mode in ("eager", "graphs"):
            _, env, alg, pool = workload(args.hist, "tf32x3", args.envs, track_episodes=track)
            env.set_obs_target(alg.storage.obs_row(0))
            w = SimpleNamespace(env=env, alg=alg, pool=pool, obs=alg.storage.obs_row(0), last=None)
            alg.cuda_graphs = mode == "graphs"
            rg = RolloutGraph(alg, env, physics=lambda t, w=w: w.env.bind_sim(**w.pool[t])) if mode == "graphs" else None
            arms[mode + ("+track" if track else "")] = dict(w=w, rg=rg, rows=[])

    def rollout(w):
        """bench.Workload.rollout: the loop RolloutGraph captures, obs_T of the previous iteration carried into storage row 0."""
        env, alg, s = w.env, w.alg, w.alg.storage
        obs = w.obs
        if obs.data_ptr() != s.obs_row(0).data_ptr():
            s.obs_row(0).copy_(obs)
            obs = s.obs_row(0)
        for t in range(s.num_transitions_per_env):
            actions = alg.act(obs, obs)
            env.bind_sim(**w.pool[t])
            env.set_obs_target(s.obs_row(t + 1))
            env.set_transition_target(s.values[t], s.rewards[t], s.dones[t], alg.gamma)
            env.pre_physics_step(actions)
            env.post_physics_step()
            obs = env.obs_buf
            alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
        return obs

    def iteration(arm, record):
        w, rg = arm["w"], arm["rg"]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        torch.cuda.synchronize()
        c0, cpu0 = counting.calls, time.process_time()
        ev[0].record()
        h0 = time.perf_counter()
        obs = rg.run(w.obs) if rg is not None else rollout(w)
        h1 = time.perf_counter()
        ev[1].record()
        w.alg.compute_returns(obs)
        ev[2].record()
        w.last = w.alg.update()
        ev[3].record()
        w.obs = obs
        torch.cuda.synchronize()
        if record:
            arm["rows"].append(dict(rollout_ms=ev[0].elapsed_time(ev[1]), gae_ms=ev[1].elapsed_time(ev[2]), update_ms=ev[2].elapsed_time(ev[3]),
                                    iteration_ms=ev[0].elapsed_time(ev[3]), host_cpu_ms=1e3 * (time.process_time() - cpu0),
                                    rollout_enqueue_ms=1e3 * (h1 - h0), library_calls=counting.calls - c0))

    for _ in range(args.warmup):
        for arm in arms.values():
            iteration(arm, False)
    info0 = gpu_info()
    for _ in range(args.runs):                          # alternating: eager, graphs[, eager+track, graphs+track], eager, ...
        for arm in arms.values():
            iteration(arm, True)
    tracker_us = {n: tracker_step_us(L, n, args.track_episodes) for n in (args.envs, 40000)} if args.track_episodes else None
    info1 = gpu_info()
    tma = tuple(bool(arm["w"].env._derived_state[:, 27].any()) for arm in arms.values())
    res = {"workload": f"bench.py flat: {args.envs} envs, history_len {args.hist}, T=40, tf32x3, 5 epochs x 4 mini-batches",
           "k1_kernel": "TMA" if all(tma) else "warp-per-env" if not any(tma) else f"differs between the arms: {tma}",
           "runs": args.runs, "warmup": args.warmup, "gpu_before": info0, "gpu_after": info1, "torch": torch.__version__}
    for name, arm in arms.items():
        rows = arm["rows"]
        res[name] = {k: dict(median=float(np.median([r[k] for r in rows])), min=float(min(r[k] for r in rows)),
                             max=float(max(r[k] for r in rows))) for k in rows[0]}
    flat = [arm["w"].alg.actor_critic.flat for arm in arms.values()]
    res["same_bits"] = all(torch.equal(flat[0], f) for f in flat[1:])
    if args.track_episodes:
        bufs = [arms[k]["w"].alg.episode_buffers() for k in ("eager+track", "graphs+track")]
        res["track_episodes"] = dict(capacity=args.track_episodes, tracker_step_us=tracker_us, same_buffers=bufs[0] == bufs[1],
                                     episodes_kept=len(bufs[0]["lenbuffer"]))
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "graph_timing.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
