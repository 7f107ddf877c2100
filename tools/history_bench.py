"""History length sweep (history_len = StateHistoryEncoder tsteps = 10, 20, 50) of the flat widowGo1 workload at 4096 envs, T = 40:

  * K1 (dwbc_post_physics_step) alone, CUDA events over back-to-back launches, with the achieved bandwidth over algorithmic bytes:
    SURVEY 8d's 10 653 B per env-step at 10 steps, of which 3 x 3 040 B are the three passes over the history row (read it, write it to
    obs, write it back shifted); at H steps those passes are 3 x H x 304 B;
  * dwbc_hist_latent over all 163 840 storage rows (the regulariser target update() computes once per iteration);
  * update() and update_dagger() (5 epochs x 4 mini-batches), and env-steps/s of whole iterations (rollout + GAE + update());
  * the card's name and power limit, read in the same run.

Prints one JSON line per history length.  Usage: python tools/history_bench.py [--precision tf32x3] [--iters 5] [--hist 10 20 50]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

N_ENVS, T = 4096, 40
K1_BYTES_H10, HIST_PASS_BYTES_PER_STEP = 10653, 3 * 76 * 4
HP = dict(value_loss_coef=1.0, use_clipped_value_loss=True, clip_param=0.2, entropy_coef=0.0, num_learning_epochs=5, num_mini_batches=4,
          learning_rate=2e-4, gamma=0.99, lam=0.95, max_grad_norm=1.0, min_policy_std=[[0.15, 0.25, 0.25] * 4 + [0.2] * 3 + [0.05] * 3],
          mixing_schedule=[1.0, 0, 1], priv_reg_coef_schedual=[0, 1, 1000, 1000])


def k1_bytes(H):
    return K1_BYTES_H10 + (H - 10) * HIST_PASS_BYTES_PER_STEP


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception:                                             # noqa: BLE001 (no nvidia-smi: the name from the driver only)
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown", max_sm_clock="unknown")


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def workload(H, precision, n_envs=N_ENVS, track_episodes=0):
    """bench.py's flat workload (same seeds, hyper-parameters and synthetic sim-state pool of T entries) at history_len H and n_envs envs:
    (params, env core, FusedPPO with its storage, pool).  track_episodes: FusedPPO's episode tracker (0: off, as in bench.py)."""
    import envstate as E
    from dwbc_b200 import synth
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.config import WidowGo1Params
    from dwbc_b200.env import FusedWidowGo1Core
    from dwbc_b200.ppo import FusedPPO
    dev = "cuda:0"
    p = WidowGo1Params(num_envs=n_envs, **dict(E.ENV_CONFIGS["flat"], history_len=H))
    st = synth.initial_env_state(p, 100)
    st.update(synth.sim_state(p, 100, 0, rp_sigma=0.05, z_lo=0.327))
    env = FusedWidowGo1Core(p, dev, state=st, seed=1000, sync_stats=False)
    env.update_command_curriculum()
    ac = FlatActorCritic(device=dev, seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=H, num_prop=76)
    alg = FusedPPO(ac, device=dev, precision=precision, track_episodes=track_episodes, **HP)
    alg.init_storage(n_envs, T, [p.num_obs], [None], [p.num_actions])
    alg.counter = 1500
    alg.generator = torch.Generator(device=dev)
    alg.generator.manual_seed(7)
    g = torch.Generator(device=dev)
    g.manual_seed(31)
    base = {k: torch.from_numpy(v).to(dev) for k, v in synth.sim_state(p, 100, 1, rp_sigma=0.05, z_lo=0.327).items()}
    pool = []
    for _ in range(T):
        s = {k: (base[k] + torch.randn(base[k].shape, device=dev, generator=g) * 0.02 * base[k].abs().clamp(min=0.05)).contiguous()
             for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]
        s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        pool.append(s)
    return p, env, alg, pool


def run(H, precision, iters):
    from dwbc_b200 import _lib as L
    p, env, alg, pool = workload(H, precision)
    ac = alg.actor_critic
    dev = "cuda:0"
    s_ = alg.storage

    def rollout():
        obs = s_.obs_row(0)
        for t in range(T):
            actions = alg.act(obs, obs)
            env.bind_sim(**pool[t])
            env.set_obs_target(s_.obs_row(t + 1))
            env.set_transition_target(s_.values[t], s_.rewards[t], s_.dones[t], alg.gamma)
            env.pre_physics_step(actions)
            env.post_physics_step()
            obs = env.obs_buf
            alg.process_env_step(env.rew_buf, env.arm_rew_buf, env.reset_buf, env.extras)
        s_.obs_row(0).copy_(obs)
        return obs

    def iteration():
        alg.compute_returns(rollout())
        alg.update()

    env.set_obs_target(s_.obs_row(0))
    iteration()                                                   # warm-up: every shape of the timed window
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        iteration()
    torch.cuda.synchronize()
    it_s = (time.perf_counter() - t0) / iters
    # K1 alone: one launch per pool entry, observations into the storage rows as in the rollout
    k = [0]

    def k1():
        t = k[0] % T
        k[0] += 1
        env.bind_sim(**pool[t])
        env.set_obs_target(s_.obs_row(t + 1))
        env.post_physics_step()
    env.set_transition_target(None)
    k1_ms = events_ms(k1, 200)
    # dwbc_hist_latent over every storage row, as update() calls it
    total = N_ENVS * T
    lld = (ac.priv_dims[-1] + 3) // 4 * 4
    zh = torch.zeros(total, lld, device=dev)
    obs_flat = s_.observations.view(total, -1)
    ws = alg._workspace(total // HP["num_mini_batches"])
    mbs = total // HP["num_mini_batches"]
    alg._set_precision()

    def latent():
        for r0 in range(0, total, mbs):
            L.check(alg._lib.dwbc_hist_latent(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs_flat[r0:]), obs_flat.stride(0), L.ptr(zh[r0:]), lld,
                                              mbs, L.ptr(ws), L.stream_ptr()), "dwbc_hist_latent")
    lat_ms = events_ms(latent, 20)

    def timed(fn):
        ms = []
        for _ in range(iters):
            rollout()
            alg.compute_returns(s_.obs_row(T))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]
    upd_ms = timed(alg.update)
    dag_ms = timed(alg.update_dagger)
    b = k1_bytes(H)
    return dict(history_len=H, num_obs=p.num_obs, precision=precision, envs=N_ENVS, rollout_steps=T,
                k1_us=round(k1_ms * 1e3, 2), k1_bytes_per_env_step=b, k1_gbps=round(N_ENVS * b / (k1_ms * 1e-3) / 1e9, 1),
                hist_latent_ms=round(lat_ms, 3), hist_latent_rows=total, update_ms=round(upd_ms, 2), update_dagger_ms=round(dag_ms, 2),
                iteration_ms=round(it_s * 1e3, 2), env_steps_per_s=round(N_ENVS * T / it_s), card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32x3", choices=["fp32", "tf32", "tf32x3"])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--hist", type=int, nargs="+", default=[10, 20, 50])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("history_bench.py measures on the GPU; no CUDA device is visible")
    for H in a.hist:
        print(json.dumps(run(H, a.precision, a.iters)), flush=True)


if __name__ == "__main__":
    main()
