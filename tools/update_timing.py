"""update() wall time (CUDA events, 3 repetitions) of the bench-sized storage."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from dwbc_b200.actor_critic import FlatActorCritic
from dwbc_b200.ppo import FusedPPO
N, T = 4096, 40
ac = FlatActorCritic(device="cuda:0", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=10, num_prop=76)
alg = FusedPPO(ac, device="cuda:0", precision=(sys.argv[1] if len(sys.argv) > 1 else "tf32"), num_learning_epochs=5, num_mini_batches=4, clip_param=0.2, gamma=0.99, lam=0.95, learning_rate=2e-4,
               mixing_schedule=[1.0, 0, 1], priv_reg_coef_schedual=[0, 1, 1000, 1000])
alg.init_storage(N, T, [860], [None], [18]); alg.counter = 1500
s = alg.storage
s._obs_all.normal_(); s.actions.normal_(); s.values.normal_(); s.returns.normal_(); s.advantages.normal_(); s.actions_log_prob.normal_().sub_(20)
alg.update(); torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3):
    alg.update()
e1.record(); torch.cuda.synchronize()
print(json.dumps({"update_ms": round(e0.elapsed_time(e1) / 3, 3)}))
