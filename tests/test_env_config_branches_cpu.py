"""The config branches no shipped config takes, on the CPU oracle alone: the rollouts of test_gpu_env_config_branches.py (same configs,
seed, start counter and steps, 1024 envs) must really take each branch, often enough that a kernel taking the other side of it fails the
GPU comparison.  The oracle is instrumented by wrapping its methods on the instance; its code is not changed.

Also the host-side bound of the collision-sample count (DwbcEnvCfg.collision_t holds 16 path samples)."""
import math

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import synth
from dwbc_b200.config import WidowGo1Params
from oracle import env_oracle as EO
from oracle import torch_utils as tu

SEED, STEPS, COUNTER0, N = 21, 30, 140, 1024      # the GPU file's rollouts: steps 141 .. 170, the push step 150 inside


class Probe:
    """An EnvOracle with wrapped methods that count, per rollout, how often each config branch decided something."""

    def __init__(self, p, o):
        self.p, self.o = p, o
        self.c = dict(term_goal_dep=0, neg_pre_clip=[0, 0], term_on_clipped=[0, 0], orn_timer=0, orn_reset=0, orn_wrap=0,
                      exhausted=0, resamples=0, resets=0, fifo_zeroed=0, push_steps=[])
        self.wins = np.zeros(10, np.int64)
        self.term_alone = np.zeros(max(1, len(p.termination_contact_indices)), np.int64)
        self._calls = None
        for name in ("_check_termination", "_compute_reward", "_term", "_resample_ee_goal", "_collision", "_push"):
            setattr(o, name, self._wrap(getattr(self, "on" + name), getattr(o, name)))

    @staticmethod
    def _wrap(hook, f):
        return lambda *a: hook(f, *a)

    # ---- termination: goal-mode dependence (WG:945-948) and the contact bodies (WG:937-963)
    def on_check_termination(self, f):
        f()
        o, p, s = self.o, self.p, self.o.s
        r, pt, _ = tu.euler_from_quat(o.root[:, 3:7])
        z_bad = o.root[:, 2] < p.term_z

        def orient(g):
            return (((r > p.term_roll) & (g[:, 2] >= 0)) | ((r < -p.term_roll) & (g[:, 2] <= 0)) |
                    ((pt > p.term_pitch) & (g[:, 1] >= 0)) | ((pt < -p.term_pitch) & (g[:, 1] <= 0)))
        cart, sph = orient(s.curr_ee_goal_cart), orient(s.curr_ee_goal_sphere)
        idx = torch.tensor(p.termination_contact_indices, dtype=torch.long)
        contact = torch.norm(o.contact_forces[:, idx, :], dim=-1) > 1.0 if len(idx) else torch.zeros(o.N, 0, dtype=torch.bool)
        other = z_bad | s.time_out_buf
        self.c["term_goal_dep"] += int(((cart | other | contact.any(1)) != (sph | other | contact.any(1))).sum())
        g = s.curr_ee_goal_cart if p.command_mode == "cart" else s.curr_ee_goal_sphere
        for b in range(contact.shape[1]):
            alone = contact[:, b] & ~contact[:, [j for j in range(contact.shape[1]) if j != b]].any(1) & ~other & ~orient(g)
            self.term_alone[b] += int(alone.sum())

    # ---- rewards: the channel sums before the positive clip (WG:170-205), rebuilt from the terms in evaluation order
    def on_compute_reward(self, f, leg_scales, arm_scales):
        self._calls = []
        f(leg_scales, arm_scales)
        calls, self._calls = self._calls, None
        i = 0
        for ch, (terms, scales) in enumerate(((self.o.leg_terms, leg_scales), (self.o.arm_terms, arm_scales))):
            buf = torch.zeros(self.o.N)
            for name in terms:
                assert calls[i][0] == name
                buf += calls[i][1] * scales[name]
                i += 1
            term = torch.zeros(self.o.N, dtype=torch.bool)
            if scales.get("termination", 0) != 0:
                assert calls[i][0] == "termination"
                term = calls[i][1] != 0
                i += 1
            self.c["neg_pre_clip"][ch] += int((buf < 0).sum())
            self.c["term_on_clipped"][ch] += int(((buf < 0) & term).sum())

    def on_term(self, f, name):
        out = f(name)
        if self._calls is not None:
            self._calls.append((name, out.clone()))
        return out

    # ---- goal resampling: orientation sites and wrap (WG:1307-1313), the winning try of the search (WG:1316-1332)
    def on_resample_ee_goal(self, f, mask, rand, col_orn, col_sph, ranges):
        if not bool(mask.any()):
            return f(mask, rand, col_orn, col_sph, ranges)
        p, s = self.p, self.o.s
        d_yaw = EO._u(rand, col_orn + 2, p.final_delta_orn[2][0], p.final_delta_orn[2][1])
        self.c["orn_timer" if col_orn == EO.RAND_GOAL_ORN else "orn_reset"] += int(mask.sum())
        self.c["orn_wrap"] += int((mask & ((d_yaw + s.base_yaw_euler[:, 2]).abs() > math.pi)).sum())
        self._todo, self._try = mask.clone(), 0
        self._won = torch.full((self.o.N,), -1, dtype=torch.long)
        f(mask, rand, col_orn, col_sph, ranges)
        self.c["resamples"] += int(mask.sum())
        self.c["exhausted"] += int((mask & (self._won < 0)).sum())
        self.wins += np.bincount(self._won[mask & (self._won >= 0)].numpy(), minlength=10)
        self._todo = None

    def on_collision(self, f, start, goal):
        hit = f(start, goal)
        if getattr(self, "_todo", None) is not None:
            won = self._todo & ~hit
            self._won[won] = self._try
            self._todo = self._todo & hit
            self._try += 1
        return hit

    def on_push(self, f, rand):
        self.c["push_steps"].append(self.o.common_step_counter)
        return f(rand)


def probe_rollout(kw, steps=STEPS):
    """The oracle over the GPU file's rollout of config `kw`; returns the Probe's counts plus the action-FIFO checks."""
    p = WidowGo1Params(num_envs=N, **kw)
    st = E.initial(p, SEED)
    o = EO.EnvOracle(p, E.oracle_state(p, st))
    pr = Probe(p, o)
    rt = E.runtime(p)
    o.common_step_counter = COUNTER0
    clipped = 0
    for t in range(1, steps + 1):
        sim = E.sim_state(p, SEED, t, o.s.env_origins)
        clipped += int((np.abs(sim["policy_actions"]) > p.clip_actions).sum())
        E.load_sim_into_oracle(o, p, sim)
        nonzero = o.s.action_history_buf.abs().amax(dim=(1, 2)) > 0
        _, _, _, rst, _ = o.post_physics_step(torch.from_numpy(synth.rand_table(p, SEED, t)), rt)
        assert not bool(o.s.action_history_buf[rst].any()), "a reset left a row of the action FIFO"
        pr.c["fifo_zeroed"] += int((rst & nonzero).sum())
        pr.c["resets"] += int(rst.sum())
    pr.c["clipped_actions"] = clipped
    return pr


@pytest.fixture(scope="module")
def probes():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = probe_rollout(E.BRANCH_CASES[name])
        return cache[name]
    return get


def test_cart_goal_decides_termination_and_orientation_resamples_wrap(probes):
    """Cart mode: the termination sign test reads the cart goal (WG:945-948 with curr_ee_goal = the cart goal) on hundreds of
    env-steps whose decision the sphere goal would flip; orientation deltas drawn at both sites, and the yaw part wraps."""
    c = probes("cart").c
    print("cart", {k: c[k] for k in ("term_goal_dep", "orn_timer", "orn_reset", "orn_wrap", "resets")})
    assert c["term_goal_dep"] >= 300
    assert c["orn_timer"] >= 30 and c["orn_reset"] >= 300 and c["orn_wrap"] >= 50


def test_positive_clip_binds_before_the_termination_term(probes):
    """only_positive_rewards (WG:170-205): the leg sum is negative before the clip on many env-steps, and the termination term is added
    to a clipped 0 on both channels."""
    c = probes("positive").c
    print("positive", {k: c[k] for k in ("neg_pre_clip", "term_on_clipped", "resets")})
    assert c["neg_pre_clip"][0] >= N and c["term_on_clipped"][0] >= 200
    assert c["neg_pre_clip"][1] >= 100 and c["term_on_clipped"][1] >= 20


@pytest.mark.parametrize("S", E.COLLISION_SAMPLES)
def test_goal_search_takes_every_try(probes, S):
    """WG:1316-1342 with S path samples: with S > 1 every try index 0..9 wins for some env and some searches use up all ten tries (the
    last try is kept); with one sample (t = 0: the start of the path) a search either passes at try 0 or never; with none, try 0 wins."""
    pr = probes(f"goals-{S}")
    w, c = pr.wins, pr.c
    print(f"goals-{S}", w.tolist(), "exhausted", c["exhausted"], "of", c["resamples"])
    assert c["resamples"] >= 1000
    if S == 0:
        assert w[0] == c["resamples"] and c["exhausted"] == 0
    elif S == 1:
        assert w[1:].sum() == 0 and w[0] >= 100 and c["exhausted"] >= 100
    else:
        assert (w >= 3).all() and c["exhausted"] >= 20


@pytest.mark.parametrize("d", E.ACTION_DELAYS)
def test_action_delay_clips_and_resets_zero_the_fifo(probes, d):
    """WG:1162-1173 at action_delay d: clip_actions 0.5 binds on most N(0, 1) actions, and resets zero the whole FIFO (WG:695-754) of envs
    whose FIFO held non-zero rows."""
    c = probes(f"delay-{d}").c
    print(f"delay-{d}", c["clipped_actions"], c["fifo_zeroed"])
    assert c["clipped_actions"] >= STEPS * N * 18 // 2
    assert c["fifo_zeroed"] >= 300


def test_raw_contact_bodies_terminate_alone_and_nothing_is_pushed(probes):
    """8 penalised and 3 termination bodies: each termination body is the only cause of some resets (so the body offsets 4 + n_penalized
    + i of the gather must be right); push_robots off: no push at step 150, while `flat`-derived configs push there."""
    pr = probes("raw")
    print("raw", pr.term_alone.tolist(), pr.c["push_steps"])
    assert (pr.term_alone >= 20).all()
    assert pr.c["push_steps"] == []
    assert probes("cart").c["push_steps"] == [150]


def test_too_many_collision_samples_raise_dwbc_error():
    """DwbcEnvCfg.collision_t holds 16 path samples: more raise DwbcError on the host (both kernels refuse them too)."""
    from dwbc_b200._lib import DwbcError
    from dwbc_b200.env import make_env_cfg
    ok = make_env_cfg(WidowGo1Params(num_envs=32, num_collision_check_samples=16), 32)
    assert ok.n_collision_samples == 16 and ok.collision_t[15] == 1.0
    for S in (17, 32, 33):
        with pytest.raises(DwbcError, match="collision"):
            make_env_cfg(WidowGo1Params(num_envs=32, num_collision_check_samples=S), 32)
    with pytest.raises(DwbcError, match="collision"):
        make_env_cfg(WidowGo1Params(num_envs=32, num_collision_check_samples=-1), 32)
