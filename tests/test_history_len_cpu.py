"""CPU: the 10-, 20- and 50-step history encoders (StateHistoryEncoder tsteps, AC:52-70) on the host side -- parameter manifest and
state_dict names against the oracle, the DwbcNetCfg geometry the library receives, and refusal of every other history length, on the
host (DwbcError) and in the library (DWBC_ERR_UNSUPPORTED, no GPU needed)."""
import contextlib
import ctypes as C
import io
import os
import sys

import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200.actor_critic import FlatActorCritic
from oracle import ppo_oracle as PO

import history_oracle as HO

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "baseline", "_ref")
# (num_hist, conv geometry (c, k, s) per conv, conv positions), restated from the table of StateHistoryEncoder
GEOMETRY = {10: (((20, 4, 2), (10, 2, 1)), (10, 4, 3)), 20: (((20, 6, 2), (10, 4, 2)), (20, 8, 3)),
            50: (((20, 8, 4), (10, 5, 1), (10, 5, 1)), (50, 11, 7, 3))}


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    return L.lib()


def make_ac(H):
    return FlatActorCritic(device="cpu", seed=0, num_priv=24, num_hist=H, num_prop=76)


@pytest.mark.parametrize("H", [10, 20, 50])
def test_manifest_and_state_dict_match_the_oracle(H):
    ac = make_ac(H)
    assert ac.manifest == HO.param_manifest(num_hist=H)
    assert ac.num_obs == 76 * (H + 1) + 24
    sd = ac.state_dict()
    convs = [n for n in sd if n.startswith("actor.history_encoder.conv_layers.")]
    cin = 30
    for k, (c, ks, _) in enumerate(GEOMETRY[H][0]):
        assert tuple(sd[f"actor.history_encoder.conv_layers.{2 * k}.weight"].shape) == (c, cin, ks)
        assert tuple(sd[f"actor.history_encoder.conv_layers.{2 * k}.bias"].shape) == (c,)
        cin = c
    assert len(convs) == 2 * len(GEOMETRY[H][0])
    assert tuple(sd["actor.history_encoder.linear_output.0.weight"].shape) == (20, 30)
    # every conv stack ends at 3 positions x 10 channels (the 30 inputs of linear_output)
    pos = [H]
    for _, ks, s in GEOMETRY[H][0]:
        pos.append((pos[-1] - ks) // s + 1)
    assert tuple(pos) == GEOMETRY[H][1]
    # the history encoder stays one contiguous block of the flat buffer (update_dagger's Adam range)
    hf, hc = ac.hist_range
    assert hf == ac.offsets["actor.history_encoder.encoder.0.weight"] and hf + hc == ac.offsets["actor.actor_backbone.0.weight"]
    ac2 = make_ac(H)
    ac2.load_state_dict(sd)
    assert all(torch.equal(ac2.views[k], sd[k]) for k in sd)


@pytest.mark.parametrize("H", [10, 20, 50])
def test_net_cfg_geometry(H):
    ac = make_ac(H)
    c, convs = ac.net_cfg, GEOMETRY[H][0]
    assert c.abi_version == L.ABI_VERSION == 5 and c.num_hist == H and c.hist_proj == 30 and c.n_hist_conv == len(convs)
    got = [(c.hist_c1, c.hist_k1, c.hist_s1), (c.hist_c2, c.hist_k2, c.hist_s2), (c.hist_c3, c.hist_k3, c.hist_s3)]
    assert got == list(convs) + [(0, 0, 0)] * (3 - len(convs))
    names = ["encoder.0", "conv_layers.0", "conv_layers.2", "conv_layers.4", "linear_output.0"]
    for i, n in enumerate(names):
        key = f"actor.history_encoder.{n}"
        if n == "conv_layers.4" and H != 50:
            assert c.off_hist_w[i] == c.off_hist_b[i] == -1
        else:
            assert c.off_hist_w[i] == ac.offsets[key + ".weight"] and c.off_hist_b[i] == ac.offsets[key + ".bias"]


def test_workspace_grows_with_the_history(lib):
    cfgs = [make_ac(H).net_cfg for H in (10, 20, 50)]
    sizes = [lib.dwbc_workspace_bytes(C.addressof(c), 4096) for c in cfgs]
    assert 0 < sizes[0] < sizes[1] < sizes[2], sizes


def test_history_oracle_is_the_oracle_at_10_steps():
    """tests/history_oracle.py restates the 20- and 50-step encoders; at 10 steps it is oracle/ppo_oracle.py, value for value, and its
    patch of the oracle leaves every oracle result unchanged."""
    from dwbc_b200 import synth
    assert HO.param_manifest(num_hist=10) == PO.param_manifest()
    assert HO.param_manifest(num_hist=10, actor_dims=(64, 32), priv_dims=(32, 16)) == PO.param_manifest(actor_dims=(64, 32), priv_dims=(32, 16))
    manifest = PO.param_manifest()
    P = {n: (torch.ones(1, 18, dtype=torch.float64) if v is None else torch.from_numpy(v).double())
         for (n, _), v in zip(manifest, synth.policy_params(manifest, 5))}
    obs = torch.from_numpy(synth.normal(5, 70, (129, 860))).double()
    z, mean = PO.hist_latent(P, obs), PO.actor_mean(P, obs, True)
    assert torch.equal(HO.hist_latent(P, obs), z)
    with HO.history_encoder():
        assert torch.equal(PO.actor_mean(P, obs, True), mean)
    assert PO.hist_latent(P, obs).equal(z)                       # restored on exit


@pytest.mark.parametrize("H", [5, 30, 100])
def test_other_history_lengths_are_refused(H):
    with pytest.raises(L.DwbcError):
        make_ac(H)
    with pytest.raises(ValueError):
        HO.param_manifest(num_hist=H)


@pytest.mark.parametrize("H", [10, 20, 50])
def test_library_refuses_a_geometry_that_does_not_match_num_hist(lib, H):
    cfg = make_ac(H).net_cfg
    assert lib.dwbc_workspace_bytes(C.addressof(cfg), 16) > 0
    other = {10: 20, 20: 50, 50: 10}[H]
    bad = []
    c = L.NetCfg.from_buffer_copy(cfg)
    c.num_hist = other                                   # the geometry of H under another num_hist
    bad.append(c)
    c = L.NetCfg.from_buffer_copy(cfg)
    c.hist_k1 += 1                                       # one kernel size off
    bad.append(c)
    c = L.NetCfg.from_buffer_copy(cfg)
    c.n_hist_conv = 5 - c.n_hist_conv                    # two convs <-> three
    bad.append(c)
    c = L.NetCfg.from_buffer_copy(cfg)
    c.hist_proj = 32
    bad.append(c)
    for c in bad:
        assert lib.dwbc_policy_act(C.addressof(c), None, None, 0, None, 0, None, None, None, None, None, 1, 0, None, None) == -2
        assert lib.dwbc_hist_latent(C.addressof(c), None, None, 0, None, 0, 1, None, None) == -2
        assert lib.dwbc_workspace_bytes(C.addressof(c), 16) < 0


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "rsl_rl")), reason="needs the unmodified rsl_rl: baseline/install_reference.sh <checkout of the reference>")
@pytest.mark.parametrize("H", [20, 50])
def test_reference_actor_critic_matches_the_oracle(H):
    """The unmodified ActorCritic(num_hist=H) against the oracle in float64: the history latent and the actor mean from it.  This pins the
    conv stacks of the table above to the reference's StateHistoryEncoder."""
    import json
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from rsl_rl.modules import ActorCritic
    from dwbc_b200 import synth
    cfg = json.load(open(os.path.join(ROOT, "baseline", "widowgo1_train_cfg.json")))
    with contextlib.redirect_stdout(io.StringIO()):
        ref = ActorCritic(76, 76, 18, **cfg["policy"], num_priv=24, num_hist=H, num_prop=76).double()
    manifest = HO.param_manifest(num_hist=H)
    assert [(n, tuple(p.shape)) for n, p in ref.named_parameters()] == [(n, tuple(s)) for n, s in manifest]
    vals = synth.policy_params(manifest, 3)
    P = {n: (torch.ones(1, 18, dtype=torch.float64) if v is None else torch.from_numpy(v).double()) for (n, _), v in zip(manifest, vals)}
    ref.load_state_dict(P, strict=True)
    obs = torch.from_numpy(synth.normal(3, 70, (257, 76 * (H + 1) + 24))).double()
    with torch.no_grad(), HO.history_encoder():
        zh = ref.actor.infer_hist_latent(obs) if hasattr(ref.actor, "infer_hist_latent") else ref.infer_hist_latent(obs)
        torch.testing.assert_close(zh, HO.hist_latent(P, obs), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref.act_inference(obs, hist_encoding=True), PO.actor_mean(P, obs, True), rtol=1e-12, atol=1e-12)
