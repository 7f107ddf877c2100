"""CPU: the evaluation surface without a GPU.  The dwbc_policy_mean binding and its host-side refusals; its chain programs (the actor
programs of dwbc_policy_act, op for op, split by head up to 2 * tiles <= SMs); EvalGraph's refusals, its observation ping-pong and the
key that decides when it re-captures."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

from dwbc_b200 import _lib as L
from test_chain_shapes_cpu import NETWORKS, describe, make_ac

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    return L.lib()


def test_binding_signature(lib):
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    decl = re.search(r"int dwbc_policy_mean\((.*?)\);", hdr, re.S).group(1)
    assert [a.strip().rsplit(" ", 1)[0] for a in decl.split(",")] == [
        "const DwbcNetCfg*", "const float*", "const float*", "int64_t", "int32_t", "float*", "int32_t", "int32_t", "void*", "dwbc_stream_t"]
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    assert L._SIGS["dwbc_policy_mean"] == [vp, vp, vp, i64, i32, vp, i32, i32, vp, vp]
    assert "dwbc_policy_mean" in L.EXPORTS and lib.dwbc_policy_mean.argtypes == L._SIGS["dwbc_policy_mean"]
    assert L.ABI_VERSION == 5


def test_host_refusals(lib):
    """NULL arguments, rows <= 0 and a bad network are refused before anything is launched."""
    ac = make_ac("S", "cpu")
    cfg, fake = C.addressof(ac.net_cfg), 1 << 40
    assert lib.dwbc_policy_mean(None, fake, fake, 860, 0, fake, 16, 0, fake, None) == -1
    for args in ((None, fake, 860, 0, fake, 16, 0, fake), (fake, None, 860, 0, fake, 16, 0, fake), (fake, fake, 860, 0, None, 16, 0, fake),
                 (fake, fake, 860, 0, fake, 16, 0, None), (fake, fake, 860, 0, fake, 0, 0, fake)):
        assert lib.dwbc_policy_mean(cfg, *args, None) == -1, args
    ac.net_cfg.activation = 99
    assert lib.dwbc_policy_mean(cfg, fake, fake, 860, 0, fake, 16, 0, fake, None) == -2


@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_chain_programs_are_the_actor_programs_of_policy_act(net):
    """what = 4 (dwbc_policy_mean) against what = 0 (dwbc_policy_act) on 132 SMs: at 33 tiles both split by head and the two mean programs
    are dwbc_policy_act's two actor programs; at 34 .. 66 tiles dwbc_policy_act shares one program per network while dwbc_policy_mean
    still splits; above, both run one actor program, the same.  Every head's last op carries the rollout hook (FIN_ACT = 1)."""
    ac = make_ac(net, "cpu")
    for precision in (2, 1):
        for hist in (0, 1):
            _, act = describe(ac, 4224, 0, hist, precision)
            npack, mean = describe(ac, 4224, 4, hist, precision)
            assert mean == [act[0], act[2]]
            assert npack == sum(len(ops) for _, ops in mean)
            assert len(describe(ac, 128 * 66, 4, hist, precision)[1]) == 2 and len(describe(ac, 128 * 66 + 1, 4, hist, precision)[1]) == 1
            _, act = describe(ac, 40960, 0, hist, precision)
            _, mean = describe(ac, 40960, 4, hist, precision)
            assert mean == [act[0]]
            assert [o["fin"] for o in mean[0][1] if o["fin"]] == [1, 1]


def test_layerwise_networks_have_no_mean_programs(lib):
    from dwbc_b200.actor_critic import FlatActorCritic
    ac = FlatActorCritic(device="cpu", num_priv=24, num_hist=10, num_prop=76, actor_hidden_dims=(512, 256, 128), critic_hidden_dims=(512, 256, 128))
    assert describe(ac, 4096, 4) == describe(ac, 4096, 0) == -2


class FakeCore:
    """The host surface of FusedWidowGo1Core that EvalGraph touches, recording what each step was given."""

    def __init__(self, N=32, num_obs=860, num_actions=18, sync_stats=False):
        self.num_envs, self.num_obs, self.num_actions, self.sync_stats = N, num_obs, num_actions, sync_stats
        self.device, self.seed, self.common_step_counter = torch.device("cpu"), 0, 0
        self._buf, self._cfg, self._args = L.EnvBuffers(), L.EnvCfg(), L.StepArgs()
        self.rew_buf = self.arm_rew_buf = torch.zeros(N)
        self.reset_buf = torch.zeros(N, dtype=torch.bool)
        self.log = []

    def set_transition_target(self, values, *a):
        self.log.append(("transition", values))

    def pre_physics_step(self, actions):
        self.log.append(("pre", actions.data_ptr()))

    def set_obs_target(self, t):
        self.obs_buf = t
        self.log.append(("obs_target", t.data_ptr()))

    def post_physics_step(self):
        self.common_step_counter += 1
        self.log.append(("post",))


def _policy(seed=0, **kw):
    from dwbc_b200.actor_critic import FlatActorCritic
    return FlatActorCritic(device="cpu", seed=seed, num_priv=24, num_prop=76, **kw)


def test_eval_graph_refusals():
    from dwbc_b200.graphs import EvalGraph
    ac, env = _policy(), FakeCore()
    for steps in (0, 3, -2, True, 4.0):
        with pytest.raises(L.DwbcError, match="steps"):
            EvalGraph(ac, env, steps)
    for cap in (0, -1, True, 2.5, "8"):
        with pytest.raises(L.DwbcError, match="track_episodes"):
            EvalGraph(ac, env, 4, track_episodes=cap)
    with pytest.raises(L.DwbcError, match="observations"):
        EvalGraph(_policy(num_hist=20), env, 4)
    with pytest.raises(L.DwbcError, match="actions"):
        EvalGraph(ac, FakeCore(num_actions=12), 4)
    with pytest.raises(L.DwbcError, match="sync_stats"):
        EvalGraph(ac, FakeCore(sync_stats=True), 4).run(torch.zeros(32, 860))


def test_ping_pong_schedule(monkeypatch):
    """Eager run (the launches a capture records): step t computes the mean of row t % 2 into the fixed action buffer, the env writes
    row (t + 1) % 2, the weight images are packed at step 0 only; obs_0 is copied into row 0 and obs_T is row 0."""
    from dwbc_b200 import graphs
    from dwbc_b200.graphs import EvalGraph
    ac, env = _policy(), FakeCore()
    ev = EvalGraph(ac, env, 6, capture=False)
    calls = []
    monkeypatch.setattr(graphs.PolicyMean, "__call__", lambda self, a, obs, out, hist, repack: calls.append((obs.data_ptr(), out.data_ptr(), repack)))
    monkeypatch.setattr(graphs.L, "lib", lambda: SimpleNamespace(dwbc_track_episodes=lambda *a: 0))
    monkeypatch.setattr(graphs.L, "ptr", lambda t, dtype=None: None if t is None else t.data_ptr())
    monkeypatch.setattr(graphs.L, "stream_ptr", lambda: None)
    obs0 = torch.randn(32, 860)
    out = ev.run(obs0)
    rows = [ev._obs[0].data_ptr(), ev._obs[1].data_ptr()]
    assert out.data_ptr() == rows[0] and torch.equal(out[:, :860], obs0)
    assert calls == [(rows[t % 2], ev._actions.data_ptr(), t == 0) for t in range(6)]
    assert [e[1] for e in env.log if e[0] == "obs_target"] == [rows[(t + 1) % 2] for t in range(6)]
    assert [e[1] for e in env.log if e[0] == "pre"] == [ev._actions.data_ptr()] * 6
    assert env.log[0] == ("transition", None) and env.common_step_counter == 6
    assert ev.run(out).data_ptr() == rows[0] and len(calls) == 12       # obs_T fed back: no copy


def test_key_changes_that_recapture(lib):
    from dwbc_b200.graphs import EvalGraph
    ac, env = _policy(), FakeCore()
    ac.net_cfg.precision = 2
    ev = EvalGraph(ac, env, 4)
    k0 = ev.key()
    ac.load_state_dict(_policy(seed=3).state_dict())          # new parameter values: replayed, not re-captured
    env.common_step_counter += 40
    assert ev.key() == k0
    ac.net_cfg.precision = 1
    assert ev.key() != k0
    ac.net_cfg.precision = 2
    assert ev.key() == k0
    env._buf.goal_state = 1 << 40                             # a new task-state tensor bound in the core
    assert ev.key() != k0
    env._buf.goal_state = None
    env._buf.obs_buf, env._buf.torques = 1 << 41, 1 << 42      # per-step targets and simulator tensors the graph sets itself
    assert ev.key() == k0
    env.seed = 5
    assert ev.key() != k0
    env.seed = 0
    env._args.generic_kernel = 1
    assert ev.key() != k0
    env._args.generic_kernel = 0
    # another EvalGraph has a workspace of its own (the key's last entry); the rest tells what else re-captures
    assert EvalGraph(ac, env, 4).key()[:-1] == k0[:-1]
    assert EvalGraph(ac, env, 4, hist_encoding=True).key()[:-1] != k0[:-1] and EvalGraph(ac, env, 6).key()[:-1] != k0[:-1]
    assert EvalGraph(ac, env, 4, track_episodes=7).key()[:-1] != k0[:-1]
    other = _policy()
    other.net_cfg.precision = 2
    assert EvalGraph(other, env, 4).key()[:-1] != k0[:-1]         # another parameter buffer
