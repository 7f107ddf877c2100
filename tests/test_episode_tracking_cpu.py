"""CPU: the episode tracker of FusedPPO(track_episodes=C) (dwbc_track_episodes, OnPolicyRunner's per-step bookkeeping OPR:140-154).
The restatement the GPU tests use as their oracle (one [N, 3] running block, the finished episodes kept as the last C rows of a
tensor) equals rsl_rl's literal deque code on random streams, bit for bit.  The entry point is exported and declared, rejects NULL
pointers and non-positive sizes without launching, and FusedPPO refuses a checkpoint whose tracker does not fit without touching
anything.  The kernel itself is tested in tests/test_gpu_episode_tracking.py."""
import ctypes
import os
import re
from collections import deque

import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200.actor_critic import FlatActorCritic
from dwbc_b200.ppo import FusedPPO
from test_oracle_golden import ppo_hp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("rewbuffer", "arm_rewbuffer", "lenbuffer")


class Restatement:
    """What dwbc_track_episodes computes: running[n] += (rew, arm_rew, 1) in fp32; the rows of the done envs, in ascending env order,
    are appended to the finished episodes, of which the last `cap` are kept; then their running rows are zeroed."""

    def __init__(self, n, cap):
        self.cap, self.running, self.rows = cap, torch.zeros(n, 3), torch.zeros(0, 3)

    def step(self, rew, arm_rew, dones):
        self.running += torch.stack([rew.float(), arm_rew.float(), torch.ones(rew.shape[0])], 1)
        ids = torch.nonzero(dones.bool())[:, 0]
        self.rows = torch.cat([self.rows, self.running[ids]])[-self.cap:]
        self.running[ids] = 0

    def buffers(self):
        return {k: self.rows[:, c].tolist() for c, k in enumerate(KEYS)}


class Literal:
    """OnPolicyRunner.learn's bookkeeping as written (OPR:140-154), with the arm channel next to the leg channel."""

    def __init__(self, n, cap):
        self.cur_reward_sum, self.cur_arm_reward_sum, self.cur_episode_length = torch.zeros(n), torch.zeros(n), torch.zeros(n)
        self.rewbuffer, self.arm_rewbuffer, self.lenbuffer = deque(maxlen=cap), deque(maxlen=cap), deque(maxlen=cap)

    def step(self, rewards, arm_rewards, dones):
        self.cur_reward_sum += rewards
        self.cur_arm_reward_sum += arm_rewards
        self.cur_episode_length += 1
        new_ids = (dones > 0).nonzero(as_tuple=False)
        self.rewbuffer.extend(self.cur_reward_sum[new_ids][:, 0].cpu().numpy().tolist())
        self.arm_rewbuffer.extend(self.cur_arm_reward_sum[new_ids][:, 0].cpu().numpy().tolist())
        self.lenbuffer.extend(self.cur_episode_length[new_ids][:, 0].cpu().numpy().tolist())
        self.cur_reward_sum[new_ids] = 0
        self.cur_arm_reward_sum[new_ids] = 0
        self.cur_episode_length[new_ids] = 0


def stream(n, steps, rate, seed, dtype=torch.bool):
    """`steps` steps of fp32 rewards of both signs over six decades, and dones at `rate` (1.0: every env, every step)."""
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        scale = 10.0 ** torch.empty(n).uniform_(-3, 3, generator=g)
        rew = torch.randn(n, generator=g) * scale
        arm = torch.randn(n, generator=g) * scale.flip(0)
        dones = (torch.rand(n, generator=g) < rate).to(dtype)
        yield rew, arm, dones


@pytest.mark.parametrize("n,cap,rate", [(1, 1, 0.5), (33, 5, 0.3), (33, 100, 1.0), (257, 7, 0.02), (1000, 100, 0.1), (64, 1000, 0.0)])
def test_restatement_equals_the_runner_deques(n, cap, rate):
    ref, lit = Restatement(n, cap), Literal(n, cap)
    for rew, arm, dones in stream(n, 60, rate, n + cap):
        ref.step(rew, arm, dones)
        lit.step(rew, arm, dones)
        assert ref.buffers() == {k: list(getattr(lit, k)) for k in KEYS}
    assert torch.equal(ref.running, torch.stack([lit.cur_reward_sum, lit.cur_arm_reward_sum, lit.cur_episode_length], 1))
    assert (len(lit.lenbuffer) == 0) == (rate == 0)


def test_entry_point_is_exported_and_declared():
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    decl = re.search(r"int dwbc_track_episodes\((.*?)\);", hdr, re.S).group(1)
    assert [p.split()[-1].lstrip("*") for p in decl.split(",")] == ["rew", "arm_rew", "dones", "num_envs", "running", "ring", "ring_pos",
                                                                    "capacity", "stream"]
    assert "dwbc_track_episodes" in L.EXPORTS and len(L._SIGS["dwbc_track_episodes"]) == 9
    assert int(re.search(r"#define DWBC_ABI_VERSION (\d+)", hdr).group(1)) == L.ABI_VERSION == 5
    assert hasattr(L.lib(), "dwbc_track_episodes")


def test_library_rejects_null_pointers_and_sizes_without_launching():
    lib = L.lib()
    p = ctypes.c_void_p(4096)                 # never dereferenced: every call below is refused before a launch
    good = [p, p, p, 8, p, p, p, 4, None]
    n0 = lib.dwbc_launch_count()
    for i in (0, 1, 2, 4, 5, 6):
        args = list(good)
        args[i] = None
        assert lib.dwbc_track_episodes(*args) == -1, i
    for n, cap in ((0, 4), (-3, 4), (8, 0), (8, -1)):
        args = list(good)
        args[3], args[7] = n, cap
        assert lib.dwbc_track_episodes(*args) == -1, (n, cap)
    assert lib.dwbc_launch_count() == n0


N, T = 4, 3


def make_alg(track=0, envs=N, seed=0, **kw):
    ac = FlatActorCritic(device="cpu", num_priv=24, num_hist=10, num_prop=76, seed=seed)
    alg = FusedPPO(ac, device="cpu", **ppo_hp(), **({"track_episodes": track} if track is not None else {}), **kw)
    alg.init_storage(envs, T, [ac.num_obs], [None], [18])
    return alg


def fill(alg, seed):
    g = torch.Generator().manual_seed(seed)
    for v in alg._episodes.values():
        v.copy_(torch.randint(0, 50, v.shape, generator=g).to(v.dtype))


def snapshot(alg):
    out = {"flat": alg.actor_critic.flat.clone(), "m": alg.optimizer.m.clone()}
    out.update({k: v.clone() for k, v in (alg._episodes or {}).items()})
    return out


def test_off_keeps_the_keys_and_buffers_of_a_ppo_built_without_it():
    plain, off = make_alg(track=None), make_alg(track=0)
    assert off._episodes is None and set(off.state_dict()) == set(plain.state_dict())
    assert {k for k, v in vars(off).items() if isinstance(v, torch.Tensor)} == {k for k, v in vars(plain).items() if isinstance(v, torch.Tensor)}
    with pytest.raises(L.DwbcError, match="track_episodes"):
        off.episode_buffers()
    for bad in (-1, 2.5, True, "100"):
        with pytest.raises(L.DwbcError, match="track_episodes"):
            make_alg(track=bad)


def test_buffers_read_the_ring_oldest_first_and_round_trip():
    alg = make_alg(track=5)
    assert alg.episode_buffers() == {k: [] for k in KEYS}
    alg._episodes["ring"].copy_(torch.arange(15, dtype=torch.float32).view(5, 3))
    alg._episodes["pos"].copy_(torch.tensor([2, 3]))                # three appended, next slot 2: slots 4, 0, 1
    assert alg.episode_buffers() == dict(rewbuffer=[12.0, 0.0, 3.0], arm_rewbuffer=[13.0, 1.0, 4.0], lenbuffer=[14.0, 2.0, 5.0])
    alg._episodes["pos"].copy_(torch.tensor([2, 17]))               # wrapped: all five, oldest at the next slot
    assert alg.episode_buffers()["rewbuffer"] == [6.0, 9.0, 12.0, 0.0, 3.0]
    fill(alg, 1)
    sd = alg.state_dict()
    assert set(sd["episodes"]) == {"running", "ring", "pos"}
    other = make_alg(track=5, seed=2)
    fill(other, 3)
    other.load_state_dict(sd)
    assert all(torch.equal(other._episodes[k], alg._episodes[k]) for k in sd["episodes"])


@pytest.mark.parametrize("case", ["on_into_off", "off_into_on", "other_envs", "other_capacity", "pos_dtype"])
def test_refused_tracker_changes_nothing(case):
    src = make_alg(track=0 if case == "off_into_on" else 8, envs=8 if case == "other_envs" else N)
    if src._episodes is not None:
        fill(src, 1)
    sd = src.state_dict()
    target = make_alg(track={"on_into_off": 0, "other_capacity": 9}.get(case, 8), seed=5)
    if target._episodes is not None:
        fill(target, 6)
    if case == "pos_dtype":
        sd["episodes"]["pos"] = sd["episodes"]["pos"].float()
    before = snapshot(target)
    with pytest.raises(L.DwbcError):
        target.load_state_dict(sd)
    after = snapshot(target)
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
