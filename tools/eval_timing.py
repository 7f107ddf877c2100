#!/usr/bin/env python
"""Evaluation costs, in one run, the arms alternating:

  * act_inference the former way (dwbc_policy_act with eps = 0, every output computed, the mean kept) against dwbc_policy_mean (the actor
    alone), at 64, 4096 and 40 960 rows, tf32x3, teacher mode, weight images packed on every call as act_inference does: CUDA events
    around --launches queued calls per sample, the mean time per call;
  * an eager evaluation loop (EvalGraph(capture=False)) against the captured one (EvalGraph.run) over 40 steps at 4096 envs on
    bench.py's flat workload (tools/history_bench.py's workload()): GPU time (CUDA events) and host enqueue time (wall clock until
    run() returns, before the synchronisation);
  * the card's name, power limit and SM clock, read before and after.

Medians, minima and maxima over --runs samples per arm (after --warmup); one JSON line, also written to --out/eval_timing.json.

    python tools/eval_timing.py [--runs 15] [--warmup 3] [--launches 50] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from graph_timing import gpu_info  # noqa: E402

STEPS, EVAL_ENVS = 40, 4096


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50, help="queued calls per inference sample")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "eval_timing.py measures on a CUDA device"
    from history_bench import workload
    from dwbc_b200 import _lib as L
    from dwbc_b200 import synth
    from dwbc_b200.graphs import EvalGraph
    lib = L.lib()

    _, env, alg, pool = workload(10, "tf32x3", EVAL_ENVS)
    ac = alg.actor_critic
    ac.net_cfg.precision = L.PRECISIONS["tf32x3"]
    na = ac.num_leg_actions + ac.num_arm_actions

    # ---- inference: the same observations through both entry points
    inf = {}
    for rows in (64, 4096, 40960):
        obs = torch.from_numpy(synth.normal(3, rows, (rows, ac.num_obs))).cuda()
        z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
        eps, act, mu, sg, val, lp, mean = z(rows, na), z(rows, na), z(rows, na), z(rows, na), z(rows, 2), z(rows, 2), z(rows, na)
        ws = z(lib.dwbc_workspace_bytes(C.addressof(ac.net_cfg), rows) // 4 + 64)

        def via_act(obs=obs, eps=eps, act=act, mu=mu, sg=sg, val=val, lp=lp, ws=ws, rows=rows):
            L.check(lib.dwbc_policy_act(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0), L.ptr(eps), 0, L.ptr(act), L.ptr(val),
                                        L.ptr(lp), L.ptr(mu), L.ptr(sg), rows, 0, L.ptr(ws), L.stream_ptr()), "dwbc_policy_act")

        def via_mean(obs=obs, mean=mean, ws=ws, rows=rows):
            L.check(lib.dwbc_policy_mean(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0), 0, L.ptr(mean), rows, 0, L.ptr(ws),
                                         L.stream_ptr()), "dwbc_policy_mean")
        inf[rows] = dict(fns=dict(policy_act=via_act, policy_mean=via_mean), ms={"policy_act": [], "policy_mean": []}, outs=(mu, mean))

    def sample_inference(rows, name, record):
        fn = inf[rows]["fns"][name]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        if record:
            inf[rows]["ms"][name].append(e0.elapsed_time(e1) / args.launches)

    # ---- evaluation: two evaluations of the same policy on the same core, eager and captured, run in turn
    ev = {mode: EvalGraph(ac, env, STEPS, track_episodes=100, physics=lambda t: env.bind_sim(**pool[t % len(pool)]), capture=mode == "graph")
          for mode in ("eager", "graph")}
    obs0 = torch.from_numpy(synth.normal(4, 1, (EVAL_ENVS, env.num_obs))).cuda().clamp(-5, 5)
    loop = {mode: dict(gpu_ms=[], enqueue_ms=[]) for mode in ev}

    def sample_eval(mode, record):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        h0 = time.perf_counter()
        ev[mode].run(obs0)
        h1 = time.perf_counter()
        e1.record()
        torch.cuda.synchronize()
        if record:
            loop[mode]["gpu_ms"].append(e0.elapsed_time(e1))
            loop[mode]["enqueue_ms"].append(1e3 * (h1 - h0))

    def round_(record):
        for rows in inf:
            for name in ("policy_act", "policy_mean"):
                sample_inference(rows, name, record)
        for mode in ev:
            sample_eval(mode, record)

    for _ in range(args.warmup):
        round_(False)
    info0 = gpu_info()
    for _ in range(args.runs):
        round_(True)
    info1 = gpu_info()
    res = {"what": f"tf32x3, teacher mode; inference: mean ms per call over {args.launches} queued calls; evaluation: {STEPS} steps at "
                   f"{EVAL_ENVS} envs, bench.py flat workload",
           "runs": args.runs, "warmup": args.warmup, "gpu_before": info0, "gpu_after": info1, "torch": torch.__version__,
           "macs_per_row": dict(actor=82944, critic=78592, history_encoder=34200)}
    for rows, d in inf.items():
        res[f"inference_{rows}"] = {k: stats(v) for k, v in d["ms"].items()}
        res[f"inference_{rows}"]["same_bits"] = bool(torch.equal(*d["outs"]))
        res[f"inference_{rows}"]["ratio_median"] = res[f"inference_{rows}"]["policy_mean"]["median"] / res[f"inference_{rows}"]["policy_act"]["median"]
    for mode, d in loop.items():
        res[f"eval_{mode}"] = {k: stats(v) for k, v in d.items()}
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "eval_timing.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
