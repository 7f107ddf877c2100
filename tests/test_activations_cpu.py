"""rsl_rl's hidden-layer activations (get_activation: elu, selu, relu, lrelu, tanh, sigmoid; crelu resolves to ReLU) without a GPU: the
derivative-from-output table of include/dwbc.h against torch autograd, the name handling of FlatActorCritic, the programs the fused chains
build for each activation (dwbc_debug_describe_chain), the library's refusal of configurations it does not implement, and -- when the
unmodified rsl_rl is installed -- that the reference applies the one activation after every hidden layer, history encoder included.

ORACLE_ACT / oracle_activation() are the float64 reference of tests/test_gpu_activations.py: oracle/ppo_oracle.py applies `F.elu` after
every hidden layer and nowhere else, so running it with that one function swapped is the reference network with another activation."""
import contextlib
import ctypes as C
import io
import os
import re
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dwbc_b200  # noqa: E402,F401
from dwbc_b200 import _lib as L  # noqa: E402
from dwbc_b200.actor_critic import FlatActorCritic  # noqa: E402
from oracle import ppo_oracle as PO  # noqa: E402
from test_chain_shapes_cpu import describe  # noqa: E402

SELU_A, SELU_S = 1.6732632423543772, 1.0507009873554805
# name -> (f(x), f'(x) as a function of y = f(x)): the table of include/dwbc.h (DwbcActivation)
ORACLE_ACT = {
    "elu": (F.elu, lambda y: torch.where(y > 0, torch.ones_like(y), y + 1)),
    "selu": (F.selu, lambda y: torch.where(y > 0, torch.full_like(y, SELU_S), y + SELU_S * SELU_A)),
    "relu": (F.relu, lambda y: (y > 0).to(y.dtype)),
    "lrelu": (lambda x: F.leaky_relu(x, 0.01), lambda y: torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01))),
    "tanh": (torch.tanh, lambda y: 1 - y * y),
    "sigmoid": (torch.sigmoid, lambda y: y * (1 - y)),
}
NEW = ["selu", "relu", "lrelu", "tanh", "sigmoid"]
# the epilogues' internal codes (gemm_simt.cuh: ACT_NONE 0, ACT_ELU 1, ACT_TANH 2, then the appended ones) that dwbc_debug_describe_chain shows
ACT_NONE, ACT_TANH = 0, 2
INTERNAL = dict(elu=1, tanh=2, selu=3, relu=4, lrelu=5, sigmoid=6)
REF = os.path.join(ROOT, "baseline", "_ref")


class _Functional:
    """torch.nn.functional with `elu` replaced"""
    def __init__(self, f):
        self.elu = f

    def __getattr__(self, name):
        return getattr(F, name)


@contextlib.contextmanager
def oracle_activation(name):
    """Run oracle/ppo_oracle.py with `name` as its hidden-layer activation."""
    saved = PO.F
    PO.F = _Functional(ORACLE_ACT[name][0])
    try:
        yield
    finally:
        PO.F = saved


def make_ac(activation, **kw):
    return FlatActorCritic(device="cpu", num_priv=24, num_hist=10, num_prop=76, activation=activation, **kw)


def test_oracle_table_matches_torch_modules_and_autograd():
    """f against the torch.nn modules rsl_rl instantiates, and f'(y) against autograd of f, in float64 on a grid through 0 and the
    tails; at x = 0 the table takes the branch torch's backward takes."""
    mods = dict(elu=nn.ELU(), selu=nn.SELU(), relu=nn.ReLU(), lrelu=nn.LeakyReLU(), tanh=nn.Tanh(), sigmoid=nn.Sigmoid())
    pts = [0.0, 1e-30, -1e-30, 1e-6, -1e-6, 1.0, -1.0, 30.0, -30.0]
    x = torch.tensor(pts + torch.linspace(-8, 8, 801, dtype=torch.float64).tolist(), dtype=torch.float64, requires_grad=True)
    for name, (f, df) in ORACLE_ACT.items():
        y = f(x)
        torch.testing.assert_close(y, mods[name](x), rtol=0, atol=0)
        (g,) = torch.autograd.grad(y.sum(), x)
        torch.testing.assert_close(df(y.detach()), g, rtol=1e-9, atol=1e-12, msg=name)


def test_activation_names_map_to_the_abi_codes():
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    body = re.search(r"enum DwbcActivation \{(.*?)\};", hdr, re.S).group(1)
    names = [t.strip().split("=")[0].strip().replace("DWBC_ACT_", "").lower() for t in body.split(",")]
    assert names == ["elu", "selu", "relu", "lrelu", "tanh", "sigmoid"]
    for code, name in enumerate(names):
        assert L.ACTIVATIONS[name] == code and make_ac(name).net_cfg.activation == code
    assert make_ac("crelu").net_cfg.activation == L.ACTIVATIONS["relu"]        # rsl_rl's get_activation('crelu') is nn.ReLU()
    with pytest.raises(L.DwbcError, match="unknown activation 'swish'.*crelu, elu, lrelu, relu, selu, sigmoid, tanh"):
        make_ac("swish")
    elu = make_ac("elu")
    for name in NEW:                                                           # no parameters: checkpoints do not depend on it
        ac = make_ac(name)
        assert ac.manifest == elu.manifest and list(ac.state_dict()) == list(elu.state_dict()) and ac.num_params == elu.num_params


def test_train_config_with_another_activation_constructs():
    import json
    from dwbc_b200 import runner_compat as RC
    from dwbc_b200.ppo import FusedPPO
    cfg = json.load(open(os.path.join(ROOT, "baseline", "widowgo1_train_cfg.json")))
    ac = RC.FusedActorCritic(76, 76, 18, **dict(cfg["policy"], activation="relu"), num_priv=24, num_hist=10, num_prop=76, device="cpu")
    assert ac.net_cfg.activation == L.ACTIVATIONS["relu"] and ac.to("cpu") is ac
    assert FusedPPO(ac, device="cpu", **cfg["algorithm"]).actor_critic.net_cfg.activation == L.ACTIVATIONS["relu"]
    with pytest.raises(L.DwbcError, match="unknown activation"):
        RC.FusedActorCritic(76, 76, 18, **dict(cfg["policy"], activation="swish"), num_priv=24, num_hist=10, num_prop=76, device="cpu")


@pytest.mark.parametrize("activation", NEW)
def test_chain_programs_carry_the_activation(activation):
    """Rollout (split per head and shared, with and without the history latent), bootstrap values, update forward and backward: the
    programs are those of ELU with every hidden op's activation replaced -- the same ops, widths and pack size, so the activation does not
    change planning -- the actor heads' outputs tanh and the critic heads' none."""
    elu, ac = make_ac("elu"), make_ac(activation)
    code = INTERNAL[activation]
    for precision in (2, 1):
        for rows, what, hist in ((4096, 0, 0), (4096, 0, 1), (16384, 0, 0), (4096, 1, 0), (40960, 2, 0), (40960, 3, 0)):
            want, got = describe(elu, rows, what, hist, precision), describe(ac, rows, what, hist, precision)
            assert got[0] == want[0] and len(got[1]) == len(want[1])
            for (nl_w, ops_w), (nl_g, ops_g) in zip(want[1], got[1]):
                assert nl_g == nl_w and len(ops_g) == len(ops_w)
                for ow, og in zip(ops_w, ops_g):
                    assert {k: v for k, v in og.items() if k != "act"} == {k: v for k, v in ow.items() if k != "act"}
                    assert og["act"] == (code if ow["act"] == INTERNAL["elu"] else ow["act"])
                    if what < 3:                                                    # forward: N = the op's output width
                        want_act = {12: ACT_TANH, 6: ACT_TANH, 1: ACT_NONE}.get(og["N"], code)   # action means, values, hidden layers
                        assert og["act"] == want_act, (rows, what, og)
            if what == 3:
                assert {o["act"] for _, ops in got[1] for o in ops} <= {code, ACT_NONE}


def test_library_refuses_unknown_activation_and_old_abi():
    """An out-of-range activation is DWBC_ERR_UNSUPPORTED and a struct of ABI version 3 (whose field was reserved) is DWBC_ERR_ARG, before
    any device work: the entry points return the code instead of running."""
    lib = L.lib()
    lib.dwbc_debug_describe_chain.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_int32]
    out = (C.c_int32 * 1024)()
    ac = make_ac("elu")
    cfg = ac.net_cfg
    cfg.precision = L.PRECISIONS["tf32x3"]                                      # (on 'fp32' no call runs on the chains)
    for bad in (6, -1, 1 << 20):
        cfg.activation = bad
        assert lib.dwbc_debug_describe_chain(C.addressof(cfg), 4096, 0, 0, 132, out, 1024) == -2
        assert lib.dwbc_policy_act(C.addressof(cfg), None, None, 0, None, 0, None, None, None, None, None, 1, 0, None, None) == -2
        assert lib.dwbc_workspace_bytes(C.addressof(cfg), 16) == -1
    cfg.activation = L.ACTIVATIONS["tanh"]
    assert lib.dwbc_debug_describe_chain(C.addressof(cfg), 4096, 0, 0, 132, out, 1024) > 0
    cfg.abi_version = 3
    assert lib.dwbc_debug_describe_chain(C.addressof(cfg), 4096, 0, 0, 132, out, 1024) == -1
    assert lib.dwbc_ppo_minibatch_grad(C.addressof(cfg), None, None, None, 1, None, None, None, None, None) == -1


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "rsl_rl")), reason="needs the unmodified rsl_rl: baseline/install_reference.sh <checkout of the reference>")
@pytest.mark.parametrize("activation", ["elu"] + NEW + ["crelu"])
def test_reference_actor_critic_matches_the_oracle(activation):
    """The unmodified ActorCritic(activation=X) against the oracle with X in float64: actor means from both latents, critic values and the
    history latent.  This pins where the reference applies the activation (every hidden layer, all four of the history encoder)."""
    import json
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from rsl_rl.modules import ActorCritic
    from rsl_rl.modules.actor_critic import get_activation
    from dwbc_b200 import synth
    if activation == "crelu":
        assert isinstance(get_activation("crelu"), nn.ReLU)
    cfg = json.load(open(os.path.join(ROOT, "baseline", "widowgo1_train_cfg.json")))
    with contextlib.redirect_stdout(io.StringIO()):
        ref = ActorCritic(76, 76, 18, **dict(cfg["policy"], activation=activation), num_priv=24, num_hist=10, num_prop=76).double()
    manifest = PO.param_manifest()
    vals = synth.policy_params(manifest, 3)
    P = {n: (torch.ones(1, 18, dtype=torch.float64) if v is None else torch.from_numpy(v).double()) for (n, _), v in zip(manifest, vals)}
    ref.load_state_dict(P, strict=True)
    obs = torch.from_numpy(synth.normal(3, 70, (257, 860))).double()
    name = "relu" if activation == "crelu" else activation
    with torch.no_grad(), oracle_activation(name):
        for hist in (False, True):
            torch.testing.assert_close(ref.act_inference(obs, hist_encoding=hist), PO.actor_mean(P, obs, hist), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref.evaluate(obs), PO.critic_values(P, obs), rtol=1e-12, atol=1e-12)
        zh = ref.actor.infer_hist_latent(obs) if hasattr(ref.actor, "infer_hist_latent") else ref.infer_hist_latent(obs)
        torch.testing.assert_close(zh, PO.hist_latent(P, obs), rtol=1e-12, atol=1e-12)
