"""Which networks run on the fused layer chains (mlp.cu: plan_chains), checked on the host without a GPU through
dwbc_debug_describe_chain.  The networks are the sweep of tests/test_gpu_chain_shapes.py; this file keeps that GPU test from silently
covering only the layer-wise path, and fails if a planner change moves one of them off the chains."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dwbc_b200  # noqa: E402,F401
from dwbc_b200.actor_critic import FlatActorCritic  # noqa: E402

# Hidden dims per network (unlisted: the shipped widowGo1 dims: priv (64, 20), actor (128,), critic (128,), leg / arm heads (128, 128)).
# num_prop 76, num_priv 24, 12 leg and 6 arm actions throughout (the oracle assumes them).
NETWORKS = {
    "S": {},                                                                       # the shipped network
    "B": dict(actor_dims=(96,), critic_dims=(64,)),                                # narrow row-major trunks feeding 128-wide heads
    "C": dict(actor_dims=(128, 68), critic_dims=(100, 36), leg_dims=(36,), arm_dims=(100, 4)),   # K / N padding, a 4-wide layer, 2-layer trunks
    "D": dict(leg_dims=(64, 32), arm_dims=(32,)),                                  # row-major head hidden layers
    "E": dict(priv_dims=(32, 16)),                                                 # latent 16
    "F": dict(actor_dims=(128, 128), leg_dims=(128, 128, 128)),                    # exactly C2_MAX_PACK weight images in the update
    "G": dict(actor_dims=(128, 128, 128), critic_dims=(128, 128, 128)),            # 38 images: the update does not fit the chains
}
# networks whose mini-batch gradient runs layer-wise although every layer fits the tile (the pack list of the update overflows)
UPDATE_OFF_CHAINS = {"G"}
_AC_KW = dict(priv_dims="priv_encoder_dims", actor_dims="actor_hidden_dims", critic_dims="critic_hidden_dims",
              leg_dims="leg_control_head_hidden_dims", arm_dims="arm_control_head_hidden_dims")
SHIPPED = dict(priv_dims=(64, 20), actor_dims=(128,), critic_dims=(128,), leg_dims=(128, 128), arm_dims=(128, 128))


def dims(net):
    """All hidden dims of a network (oracle.ppo_oracle.param_manifest keywords)."""
    return dict(SHIPPED, **NETWORKS[net])


def make_ac(net, device):
    return FlatActorCritic(device=device, num_priv=24, num_hist=10, num_prop=76, **{_AC_KW[k]: v for k, v in NETWORKS[net].items()})


def describe(ac, rows, what, hist=0, precision=2, sms=132):
    """dwbc_debug_describe_chain -> (pack items, [(n_loads, [op dict])]) or the negative error code."""
    from dwbc_b200 import _lib as L
    lib = L.lib()
    lib.dwbc_debug_describe_chain.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_int32]
    ac.net_cfg.precision = precision
    out = (C.c_int32 * 1024)()
    k = lib.dwbc_debug_describe_chain(C.addressof(ac.net_cfg), rows, what, hist, sms, out, 1024)
    if k < 0:
        return k
    v, i, progs = list(out[:k]), 2, []
    for _ in range(v[0]):
        n_ops, n_loads = v[i], v[i + 1]
        i += 2
        progs.append((n_loads, [dict(zip(("N", "kpad", "act", "fin", "fin_c", "out_col0", "y", "y_img"), v[i + 8 * j:i + 8 * j + 8]))
                                for j in range(n_ops)]))
        i += 8 * n_ops
    assert i == k
    return v[1], progs


@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_sweep_networks_run_on_the_chains(net):
    """Rollout (split into one program per head at 4 * 33 tiles <= 132 SMs, shared above), bootstrap values and the mini-batch update
    (forward + loss, backward) of every sweep network on both tensor-core precisions: on the chains, except the update of G.  The programs
    hold every layer of the network in order (update forward: encoder, backbone, leg head + 12, arm head + 6; critic: backbone, heads + 1),
    each hidden activation the backward pass reads is stored, and it is a tile image exactly when it is 128 wide."""
    d = dims(net)
    ac = make_ac(net, "cpu")
    for precision in (2, 1):
        npack, progs = describe(ac, 4224, 0, precision=precision)
        assert len(progs) == 4 and npack <= 36
        assert len(describe(ac, 4225, 0, precision=precision)[1]) == 2
        assert len(describe(ac, 4224, 0, hist=1, precision=precision)[1]) == 4
        assert len(describe(ac, 4224, 1, precision=precision)[1]) == 2
        fwd, bwd = describe(ac, 16973, 2, precision=precision), describe(ac, 16973, 3, precision=precision)
        if net in UPDATE_OFF_CHAINS:
            assert fwd == bwd == -2
            continue
        assert fwd[0] == bwd[0] <= 36
        (_, actor), (_, critic) = fwd[1]
        assert [o["N"] for o in actor] == list(d["priv_dims"]) + list(d["actor_dims"]) + list(d["leg_dims"]) + [12] + list(d["arm_dims"]) + [6]
        assert [o["N"] for o in critic] == list(d["critic_dims"]) + list(d["leg_dims"]) + [1] + list(d["arm_dims"]) + [1]
        hidden = [o for o in actor + critic if o["fin"] == 0]
        assert all(o["y"] == 1 and o["y_img"] == (o["N"] == 128) for o in hidden)
    assert describe(ac, 16973, 2, precision=0) == -2                    # fp32: the layer-wise anchor


def test_update_pack_list_at_its_limit():
    """The update packs one weight image per forward and per backward op: 30 for the shipped network, exactly C2_MAX_PACK = 36 for F (on
    the chains).  G would need 38 (two more 128-wide backbone layers per network than the shipped one) and runs layer-wise."""
    assert describe(make_ac("F", "cpu"), 16973, 2)[0] == 36
    assert describe(make_ac("S", "cpu"), 16973, 2)[0] == 30
