"""TEST INFRASTRUCTURE ONLY -- the 20- and 50-step branches of StateHistoryEncoder (AC:39-84), which oracle/ppo_oracle.py does not
restate (it keeps the tsteps == 10 branch, AC:57-62).  The conv stacks by tsteps are tabled once here (HIST_CONVS); the 10-step row is the
oracle's own, and tests/test_history_len_cpu.py checks that this module reproduces the oracle there exactly.

`history_encoder()` runs oracle/ppo_oracle.py with the history encoder of this module, the way test_activations_cpu.oracle_activation()
swaps its activation: PPO.act, PPO.update and update_dagger of the oracle then use the encoder whose tsteps the parameters P hold."""
import contextlib

import torch.nn.functional as F

from oracle import ppo_oracle as PO

# tsteps -> (out_channels, kernel, stride) of conv_layers.0, .2 (, .4) (AC:52-70); every stack ends at 3 positions x 10 channels, the
# 30 inputs of linear_output
HIST_CONVS = {10: ((20, 4, 2), (10, 2, 1)), 20: ((20, 6, 2), (10, 4, 2)), 50: ((20, 8, 4), (10, 5, 1), (10, 5, 1))}
PREFIX = "actor.history_encoder."


def param_manifest(num_hist=10, **kw):
    """oracle.param_manifest with the history encoder of `num_hist` steps; any other tsteps raises, as the reference does (AC:69)."""
    if num_hist not in HIST_CONVS:
        raise ValueError(f"tsteps = {num_hist} not implemented")
    base = PO.param_manifest(**kw)
    first = next(i for i, (n, _) in enumerate(base) if n.startswith(PREFIX))
    last = max(i for i, (n, _) in enumerate(base) if n.startswith(PREFIX))
    latent, num_prop = base[last][1][0], base[first][1][1]
    enc = [(PREFIX + "encoder.0.weight", (30, num_prop)), (PREFIX + "encoder.0.bias", (30,))]
    cin = 30
    for k, (co, ks, _) in enumerate(HIST_CONVS[num_hist]):
        enc += [(PREFIX + f"conv_layers.{2 * k}.weight", (co, cin, ks)), (PREFIX + f"conv_layers.{2 * k}.bias", (co,))]
        cin = co
    enc += [(PREFIX + "linear_output.0.weight", (latent, 3 * cin)), (PREFIX + "linear_output.0.bias", (latent,))]
    return base[:first] + enc + base[last + 1:]


def num_steps(P):
    """tsteps of the history encoder in P, told apart by its first conv's kernel size (one per row of HIST_CONVS)."""
    k = P[PREFIX + "conv_layers.0.weight"].shape[-1]
    return next(t for t, convs in HIST_CONVS.items() if convs[0][1] == k)


def hist_latent(P, obs, num_prop=76):
    """actor.infer_hist_latent (AC:223-225) with the encoder of P's tsteps (AC:79-84)."""
    T = num_steps(P)
    h = obs[:, -T * num_prop:].reshape(-1, T, num_prop)
    nd = h.shape[0]
    x = F.elu(F.linear(h.reshape(nd * T, -1), P[PREFIX + "encoder.0.weight"], P[PREFIX + "encoder.0.bias"]))     # AC:80
    x = x.reshape(nd, T, -1).permute(0, 2, 1)
    for k, (_, _, stride) in enumerate(HIST_CONVS[T]):                                                            # AC:81
        x = F.elu(F.conv1d(x, P[PREFIX + f"conv_layers.{2 * k}.weight"], P[PREFIX + f"conv_layers.{2 * k}.bias"], stride=stride))
    return F.elu(F.linear(x.flatten(1), P[PREFIX + "linear_output.0.weight"], P[PREFIX + "linear_output.0.bias"]))  # AC:82-83


@contextlib.contextmanager
def history_encoder():
    """Run oracle/ppo_oracle.py with hist_latent above.  Its callers pass the oracle's default num_hist = 10; the steps come from P."""
    saved = PO.hist_latent
    PO.hist_latent = lambda P, obs, num_prop=76, num_hist=None: hist_latent(P, obs, num_prop)
    try:
        yield
    finally:
        PO.hist_latent = saved
