"""Micro-benchmark of the fused post-physics kernel alone (CUDA events, rotating sim-state pool > L2)."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import envstate as E
from dwbc_b200 import synth
from dwbc_b200.env import FusedWidowGo1Core

def main(name="flat", N=4096, iters=200, pool_n=40):
    p = E.make_params(name, N)
    st = synth.initial_env_state(p, 100); st.update(synth.sim_state(p, 100, 0, rp_sigma=0.05, z_lo=0.327))
    if p.measure_heights: st["height_samples"] = synth.height_field(p, 100)
    env = FusedWidowGo1Core(p, "cuda:0", state=st, seed=1, sync_stats=False, generic_kernel=bool(os.environ.get("DWBC_ENV_KERNEL_V1"))); env.update_command_curriculum()
    base = {k: torch.from_numpy(v).cuda() for k, v in synth.sim_state(p, 100, 1, rp_sigma=0.05, z_lo=0.327).items()}
    pool = []
    for t in range(pool_n):
        s = {k: (base[k] * (1 + 0.01 * torch.randn_like(base[k]))).contiguous() for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]; s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        pool.append(s)
    obs = torch.zeros(pool_n + 1, N, p.num_obs, device="cuda")
    def step(t):
        env.bind_sim(**pool[t % pool_n]); env.set_obs_target(obs[t % pool_n]); env.post_physics_step()
    for t in range(20): step(t)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for t in range(iters):
        env._stats.zero_()
        ev[t][0].record(); 
        env.bind_sim(**pool[t % pool_n]); env.set_obs_target(obs[t % pool_n])
        env.common_step_counter += 1
        a = env._args; a.rand_uniform = None; a.seed, a.step = env.seed, env.common_step_counter; a.do_push = 0
        import ctypes as C
        from dwbc_b200 import _lib as L
        L.check(env._lib.dwbc_post_physics_step(C.addressof(env._cfg), C.addressof(env._buf), C.addressof(a), L.stream_ptr()), "k1")
        ev[t][1].record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) * 1e3 for a, b in ev)
    med = ts[len(ts) // 2]
    print(json.dumps(dict(kernel="v1" if os.environ.get("DWBC_ENV_KERNEL_V1") else "v2", config=name, N=N, us_median=med, us_min=ts[0], us_p90=ts[int(.9 * len(ts))],
                          gbps=N * 10653 / med / 1e3, resets=int(env.reset_buf.sum()))))
if __name__ == "__main__":
    main(*(sys.argv[1:2] or ["flat"]), N=int(sys.argv[2]) if len(sys.argv) > 2 else 4096)


def queued(name="flat", N=4096, n=40, reps=5):
    """True back-to-back kernel time: fill the stream behind a ~20 ms spin kernel, then time n launches."""
    import ctypes as C
    from dwbc_b200 import _lib as L
    p = E.make_params(name, N)
    st = synth.initial_env_state(p, 100); st.update(synth.sim_state(p, 100, 0, rp_sigma=0.05, z_lo=0.327))
    if p.measure_heights: st["height_samples"] = synth.height_field(p, 100)
    env = FusedWidowGo1Core(p, "cuda:0", state=st, seed=1, sync_stats=False, generic_kernel=bool(os.environ.get("DWBC_ENV_KERNEL_V1"))); env.update_command_curriculum()
    base = {k: torch.from_numpy(v).cuda() for k, v in synth.sim_state(p, 100, 1, rp_sigma=0.05, z_lo=0.327).items()}
    pool = []
    for t in range(n):
        s = {k: (base[k] * (1 + 0.01 * torch.randn_like(base[k]))).contiguous() for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]; s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        pool.append(s)
    obs = torch.zeros(n, N, p.num_obs, device="cuda")
    for t in range(n): env.bind_sim(**pool[t]); env.set_obs_target(obs[t]); env.post_physics_step()
    res = []
    for r in range(reps):
        torch.cuda.synchronize()
        torch.cuda._sleep(40_000_000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for t in range(n):
            env.bind_sim(**pool[t]); env.set_obs_target(obs[t])
            env.common_step_counter += 1
            a = env._args; a.rand_uniform = None; a.seed, a.step = env.seed, env.common_step_counter; a.do_push = 0
            L.check(env._lib.dwbc_post_physics_step(C.addressof(env._cfg), C.addressof(env._buf), C.addressof(a), L.stream_ptr()), "k1")
        e1.record(); torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) * 1e3 / n)
    us = sorted(res)[len(res) // 2]
    print(json.dumps(dict(kernel="v1" if os.environ.get("DWBC_ENV_KERNEL_V1") else "v2", config=name, N=N, us_per_launch=us, all=res, gbps=N * 10653 / us / 1e3, frac_of_datasheet_3350_gbs=N * 10653 / us / 1e3 / 3350)))

if __name__ == "__main__" and len(sys.argv) > 3 and sys.argv[3] == "queued":
    queued(sys.argv[1], int(sys.argv[2]))
