"""Where the time of update() and act() goes at the bench shapes (4096 envs x 40 steps, 5 epochs x 4 mini-batches), per precision:

  (a) update() ms from CUDA events: REPS sets of N_UPD back-to-back calls after a warm-up (median, min, max over the sets);
  (b) in a separate pass, torch.profiler (CUDA activities) over two update() calls and 40 act() calls: launches, total us and share
      per kernel name.

Each library named with --lib is measured in subprocesses of its own, alternating (A B A B ...) so that a drift of the machine hits
both alike; the card's name and power limit are read in the same call.  One JSON file per subprocess goes to --out, the summary is
printed.  Needs a GPU: there is no fallback.

  python tools/update_breakdown.py --out bench_out/breakdown                                  # the built library
  python tools/update_breakdown.py --out bench_out/ab --lib old/libdwbc.so --lib new/libdwbc.so --rounds 2
  python tools/update_breakdown.py --out bench_out/relu --activation relu                     # another hidden-layer activation
"""
import argparse, json, os, re, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_ENVS, T_STEPS, N_UPD, REPS, N_ACT = 4096, 40, 10, 5, 40


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def short(name):
    """Kernel name without return type, namespaces and argument list (template arguments stay: they tell the instantiations apart)."""
    name = re.sub(r"\(.*$", "", name)
    return re.sub(r"^(void |at::native::|dwbc::|\(anonymous namespace\)::)+", "", name)[:96]


def child(a):
    sys.path.insert(0, ROOT)
    import torch
    from dwbc_b200 import _lib
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib[0])          # before the first _lib.lib()
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("update_breakdown needs a CUDA device")
    res = {"lib": _lib.LIB_PATH, "activation": a.activation, "card": card(), "torch": torch.__version__, "precisions": {}}
    for prec in a.precisions:
        ac = FlatActorCritic(device="cuda:0", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=10, num_prop=76,
                             activation=a.activation)
        alg = FusedPPO(ac, device="cuda:0", precision=prec, num_learning_epochs=5, num_mini_batches=4, clip_param=0.2, gamma=0.99, lam=0.95,
                       learning_rate=2e-4, mixing_schedule=[1.0, 0, 1], priv_reg_coef_schedual=[0, 1, 1000, 1000])
        alg.init_storage(N_ENVS, T_STEPS, [860], [None], [18]); alg.counter = 1500
        s = alg.storage
        s._obs_all.normal_(); s.actions.normal_(); s.values.normal_(); s.returns.normal_(); s.advantages.normal_(); s.actions_log_prob.normal_().sub_(20)
        obs = s.observations[0]
        for _ in range(2):
            alg.update()
        alg.act(obs, obs, False)
        torch.cuda.synchronize()
        sets = []
        for _ in range(REPS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(N_UPD):
                alg.update()
            e1.record(); torch.cuda.synchronize()
            sets.append(e0.elapsed_time(e1) / N_UPD)
        # act(): N_ACT back-to-back calls (host launch cost included, as in a rollout)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(N_ACT):
            alg.act(obs, obs, False)
        e1.record(); torch.cuda.synchronize()
        act_ms = e0.elapsed_time(e1) / N_ACT
        kern = {}
        for tag, fn, n in (("update", alg.update, 2), ("act", lambda: alg.act(obs, obs, False), N_ACT)):
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(n):
                    fn()
                torch.cuda.synchronize()
            rows = [(short(e.key), e.count, e.device_time_total) for e in p.key_averages() if e.device_time_total > 0]
            tot = sum(r[2] for r in rows) or 1.0
            kern[tag] = {"calls": n, "gpu_us_total": tot,
                         "kernels": [dict(name=k, launches=c, us=round(us, 1), share=round(us / tot, 4)) for k, c, us in sorted(rows, key=lambda r: -r[2])]}
        res["precisions"][prec] = {"update_ms_sets": [round(x, 3) for x in sets], "update_ms_median": round(statistics.median(sets), 3),
                                   "update_ms_min": round(min(sets), 3), "update_ms_max": round(max(sets), 3), "act_ms": round(act_ms, 4), "profile": kern}
        del alg, ac
    with open(a.child, "w") as f:
        json.dump(res, f, indent=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory (one JSON per subprocess + summary.json)")
    ap.add_argument("--lib", action="append", default=[], help="libdwbc.so to measure; repeat to compare (default: the built one)")
    ap.add_argument("--rounds", type=int, default=1, help="times each library is measured (alternating)")
    ap.add_argument("--precisions", nargs="+", default=["tf32x3", "tf32"], choices=["tf32x3", "tf32"])
    ap.add_argument("--activation", default="elu", help="hidden-layer activation of the network (rsl_rl name)")
    ap.add_argument("--top", type=int, default=8, help="kernels listed per table")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)
    os.makedirs(a.out, exist_ok=True)
    libs = a.lib or [None]
    runs = []
    for rnd in range(a.rounds):
        for li, lib in enumerate(libs):
            path = os.path.join(a.out, f"run_r{rnd}_lib{li}.json")
            cmd = [sys.executable, os.path.abspath(__file__), "--out", a.out, "--child", path, "--precisions", *a.precisions, "--activation", a.activation] + (["--lib", lib] if lib else [])
            subprocess.run(cmd, check=True)                # no GPU / a failing library: the whole command fails
            runs.append((li, json.load(open(path))))
    print("card (name, power limit, max SM clock):", runs[0][1]["card"], "| activation:", a.activation)
    summary = {"card": runs[0][1]["card"], "activation": a.activation, "libs": [l or "built" for l in libs], "update_ms": {}}
    for prec in a.precisions:
        for li, lib in enumerate(libs):
            sets = [x for i, r in runs if i == li for x in r["precisions"][prec]["update_ms_sets"]]
            acts = [r["precisions"][prec]["act_ms"] for i, r in runs if i == li]
            summary["update_ms"][f"{prec} lib{li}"] = dict(median=statistics.median(sets), min=min(sets), max=max(sets), sets=len(sets), act_ms=acts)
            print(f"{prec:7s} lib{li} ({lib or 'built'}): update() {statistics.median(sets):.2f} ms median [{min(sets):.2f}, {max(sets):.2f}] over {len(sets)} sets "
                  f"of {N_UPD}; act() {', '.join('%.3f' % x for x in acts)} ms")
        for li, lib in enumerate(libs):
            first = next(r for i, r in runs if i == li)["precisions"][prec]["profile"]
            for tag in ("update", "act"):
                t = first[tag]
                print(f"  {prec} lib{li} {tag} x{t['calls']}: {t['gpu_us_total'] / t['calls']:.0f} us of GPU time per call")
                for k in t["kernels"][:a.top]:
                    print(f"    {k['share'] * 100:5.1f} %  {k['us'] / t['calls']:9.1f} us/call  {k['launches'] // t['calls']:4d} launches/call  {k['name']}")
    with open(os.path.join(a.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
