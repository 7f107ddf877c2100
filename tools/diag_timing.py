#!/usr/bin/env python
"""Cost of the PPO update diagnostics, in one run, the arms alternating:

  * update() of bench.py's sizes (4096 envs x 40 steps, 5 epochs x 4 mini-batches of 40 960 rows) with diagnostics off, in this tree and
    in a second tree given by --baseline (the library before the diagnostics, built in place there), and with diagnostics on in this
    tree: CUDA events around --updates update() calls per sample.  The update's rollout storage is refilled from the same seeded
    normals before each sample, so every arm runs the same numbers;
  * whether the arms compute the same: a hash of the parameters, both Adam moments and the returned losses after the first update(),
    which must agree between every arm;
  * the card's name, power limit and SM clock, read before and after.

Each arm lives in a worker process of its own tree (the two trees' packages share a name); the parent process alternates them.  Medians,
minima and maxima over --runs samples per arm (after --warmup); one JSON line, also written to --out/diag_timing.json.

--profile instead runs one update() of this tree with diagnostics off and one with them on under torch.profiler (CUDA activity, after a
warm-up update) and reports the device time per kernel name summed over the update, and the difference on - off per kernel: where the
cost of the diagnostics goes.  A run of its own, since tracing slows the host; written to --out/diag_profile.json.

    python tools/diag_timing.py --baseline DIR [--precisions tf32x3,fp32] [--runs 9] [--warmup 2] [--updates 3] [--out DIR]
    python tools/diag_timing.py --profile [--precisions tf32x3] [--out DIR]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, T = 4096, 40


def worker(tree, precision, diagnostics, updates, profile=False):
    """One arm: reads a line per sample from stdin, answers with the mean update() time in ms (first line: the result hash)."""
    sys.path.insert(0, tree)
    import torch
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cuda:0", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=10, num_prop=76)
    kw = dict(diagnostics=True) if diagnostics else {}
    alg = FusedPPO(ac, device="cuda:0", precision=precision, num_learning_epochs=5, num_mini_batches=4, clip_param=0.2, gamma=0.99,
                   lam=0.95, learning_rate=2e-4, mixing_schedule=[1.0, 0, 1], priv_reg_coef_schedual=[0, 1, 1000, 1000], **kw)
    alg.init_storage(N, T, [860], [None], [18])
    alg.counter = 1500
    s = alg.storage
    g = torch.Generator(device="cuda:0")

    def fill():
        g.manual_seed(5)
        for t in (s._obs_all, s.actions, s.values, s.returns, s.advantages, s.actions_log_prob, s.mu):
            t.normal_(generator=g)
        s.actions_log_prob.sub_(20.0)
        s.sigma.uniform_(0.8, 1.2, generator=g)
        s.mu.clamp_(-0.9, 0.9)
    perm = torch.randperm(N * T, device="cuda:0", generator=torch.Generator(device="cuda:0").manual_seed(9))
    fill()
    losses = alg.update(indices=perm)
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for t in (ac.flat, alg.optimizer.m, alg.optimizer.v):
        h.update(t.cpu().numpy().tobytes())
    h.update(repr(losses).encode())
    print(json.dumps(dict(hash=h.hexdigest()[:16])), flush=True)
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        fill()
        alg.update(indices=perm)
        fill()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as pr:
            alg.update(indices=perm)
            torch.cuda.synchronize()
        us = {}
        for e in pr.key_averages():
            if e.device_type.name == "CUDA" and getattr(e, "self_device_time_total", 0) > 0:
                us[e.key[:60]] = us.get(e.key[:60], 0.0) + e.self_device_time_total
        print(json.dumps(dict(kernel_us=us)), flush=True)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in sys.stdin:
        fill()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(updates):
            alg.update(indices=perm)
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps(dict(ms=e0.elapsed_time(e1) / updates)), flush=True)
        if diagnostics:
            alg.update_diagnostics()


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.strip().splitlines()[0].split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default=None, help="tree of the library without diagnostics (libdwbc.so built in place)")
    ap.add_argument("--profile", action="store_true", help="per-kernel device time of one update, diagnostics off and on")
    ap.add_argument("--precisions", default="tf32x3,fp32")
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--updates", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=3, metavar=("TREE", "PRECISION", "DIAG"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(os.path.abspath(a.worker[0]), a.worker[1], a.worker[2] == "1", a.updates, a.profile)
    import numpy as np
    if a.profile:
        res = dict(gpu=gpu_info())
        for p in a.precisions.split(","):
            k = {}
            for name, diag in (("off", 0), ("on", 1)):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", ROOT, p, str(diag), "--profile"], capture_output=True,
                                     text=True, cwd=ROOT, check=True).stdout.strip().splitlines()
                k[name] = json.loads(out[-1])["kernel_us"]
            diff = {n: k["on"].get(n, 0.0) - k["off"].get(n, 0.0) for n in set(k["on"]) | set(k["off"])}
            res[p] = dict(total_us_off=sum(k["off"].values()), total_us_on=sum(k["on"].values()),
                          on_minus_off_us=dict(sorted(((n, v) for n, v in diff.items() if abs(v) >= 1.0), key=lambda x: -abs(x[1]))))
        line = json.dumps(res)
        print(line)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "diag_profile.json"), "w") as f:
                f.write(line + "\n")
        return
    if a.baseline is None:
        ap.error("--baseline is required (or --profile)")
    info0 = gpu_info()
    arms = {}
    for p in a.precisions.split(","):
        for name, tree, diag in (("baseline_off", a.baseline, 0), ("off", ROOT, 0), ("on", ROOT, 1)):
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", os.path.abspath(tree), p, str(diag), "--updates", str(a.updates),
                   "--baseline", a.baseline]
            proc = subprocess.Popen(cmd, stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True, cwd=tree)
            arms[(p, name)] = dict(proc=proc, hash=json.loads(proc.stdout.readline())["hash"], ms=[])
    for r in range(a.warmup + a.runs):
        for arm in arms.values():
            arm["proc"].stdin.write("go\n")
            arm["proc"].stdin.flush()
            ms = json.loads(arm["proc"].stdout.readline())["ms"]
            if r >= a.warmup:
                arm["ms"].append(ms)
    for arm in arms.values():
        arm["proc"].stdin.close()
        arm["proc"].wait()
    res = dict(gpu_before=info0, gpu_after=gpu_info(), rows_per_minibatch=N * T // 4, minibatches=20, updates_per_sample=a.updates)
    for p in a.precisions.split(","):
        d = {name: dict(median=float(np.median(arms[(p, name)]["ms"])), min=min(arms[(p, name)]["ms"]), max=max(arms[(p, name)]["ms"]),
                        hash=arms[(p, name)]["hash"]) for name in ("baseline_off", "off", "on")}
        d["same_results"] = len({v["hash"] for v in d.values()}) == 1
        d["on_minus_off_ms"] = d["on"]["median"] - d["off"]["median"]
        res[p] = d
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "diag_timing.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
