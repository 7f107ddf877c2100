#!/usr/bin/env python
"""Eager against CUDA-graph replay on bench.py's flat workload (T = 40, tf32x3, 5 epochs x 4 mini-batches) at --hist history steps and
--envs envs (default 10 and 4096: bench.py's own workload; built by tools/history_bench.py's workload()).

Two workloads from the same seeds, one eager and one with a captured rollout (dwbc_b200.graphs.RolloutGraph) and captured update()
(FusedPPO(cuda_graphs=True)), run one iteration each in turn, --runs times (after --warmup iterations each).  Per iteration it records
the rollout, update() and whole-iteration times (CUDA events), the host CPU time of the process (time.process_time; it includes the time
the host waits in the iteration's one synchronisation), the host wall time spent enqueueing the rollout, and the library calls made
through the ctypes binding.  Which post-physics kernel ran is read from derived_state column 27 (the TMA kernel's out-of-range history
counter; the warp-per-env kernel leaves it at 0).  The card's name, power limit and clocks are read in the same run.

    python tools/graph_timing.py [--hist 10] [--envs 4096] [--runs 5] [--warmup 3] [--out DIR]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hist", type=int, default=10, choices=[10, 20, 50], help="history_len (StateHistoryEncoder tsteps)")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "graph_timing.py measures on a CUDA device"
    from history_bench import workload
    from dwbc_b200 import _lib as L
    from dwbc_b200.graphs import RolloutGraph
    counting = CountingLib(L.lib())
    L._lib = counting                                   # FusedPPO / the env core / the storage bind L.lib() at construction

    arms = {}
    for name in ("eager", "graphs"):
        _, env, alg, pool = workload(args.hist, "tf32x3", args.envs)
        env.set_obs_target(alg.storage.obs_row(0))
        w = SimpleNamespace(env=env, alg=alg, pool=pool, obs=alg.storage.obs_row(0), last=None)
        alg.cuda_graphs = name == "graphs"
        rg = RolloutGraph(alg, env, physics=lambda t, w=w: w.env.bind_sim(**w.pool[t])) if name == "graphs" else None
        arms[name] = dict(w=w, rg=rg, rows=[])

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
    for _ in range(args.runs):                          # alternating: eager, graphs, eager, ...
        for arm in arms.values():
            iteration(arm, True)
    info1 = gpu_info()
    tma = tuple(bool(arm["w"].env._derived_state[:, 27].any()) for arm in arms.values())
    res = {"workload": f"bench.py flat: {args.envs} envs, history_len {args.hist}, T=40, tf32x3, 5 epochs x 4 mini-batches",
           "k1_kernel": {(True, True): "TMA", (False, False): "warp-per-env"}.get(tma, f"differs between the arms: {tma}"),
           "runs": args.runs, "warmup": args.warmup, "gpu_before": info0, "gpu_after": info1, "torch": torch.__version__}
    for name, arm in arms.items():
        rows = arm["rows"]
        res[name] = {k: dict(median=float(np.median([r[k] for r in rows])), min=float(min(r[k] for r in rows)),
                             max=float(max(r[k] for r in rows))) for k in rows[0]}
    res["same_bits"] = bool(torch.equal(arms["eager"]["w"].alg.actor_critic.flat, arms["graphs"]["w"].alg.actor_critic.flat))
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "graph_timing.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
