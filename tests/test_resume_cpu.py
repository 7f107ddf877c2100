"""FusedPPO.state_dict() / load_state_dict() on the host: what a checkpoint restores (parameters, both Adam states, `counter`, the
generator the algorithm draws from), that it survives torch.save / torch.load with the default weights_only loader, and what it
refuses (a save in the middle of a rollout, another network, another storage shape, an unknown format version) without touching
anything.  The GPU run that resumes training bit for bit is tests/test_gpu_resume.py."""
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200.actor_critic import FlatActorCritic
from dwbc_b200.ppo import FusedPPO
from test_oracle_golden import ppo_hp

N, T = 4, 3


def make_alg(num_hist=10, actor_hidden_dims=(128,), envs=N, seed=0):
    ac = FlatActorCritic(device="cpu", num_priv=24, num_hist=num_hist, num_prop=76, actor_hidden_dims=actor_hidden_dims, seed=seed)
    alg = FusedPPO(ac, device="cpu", **ppo_hp())
    alg.init_storage(envs, T, [ac.num_obs], [None], [18])
    alg.generator = torch.Generator().manual_seed(100 + seed)
    return alg


def train_like(alg, seed):
    """Give every piece of state a value no fresh object has: parameters, both Adam states, counter, generator position."""
    g = torch.Generator().manual_seed(seed)
    ac = alg.actor_critic
    ac.flat.copy_(ac.flat_from({n: torch.randn(s, generator=g) for n, s in ac.manifest}))
    for opt, step in ((alg.optimizer, 7), (alg.hist_encoder_optimizer, 3)):
        um, uv = ac.unflat(opt.m), ac.unflat(opt.v)
        for n in opt._names():
            um[n].normal_(generator=g)
            uv[n].uniform_(generator=g)
        opt.step = step
    alg.counter = 1502
    torch.randperm(40, generator=alg.generator)


def snapshot(alg):
    ac = alg.actor_critic
    return dict(flat=ac.flat.clone(), m=alg.optimizer.m.clone(), v=alg.optimizer.v.clone(), hm=alg.hist_encoder_optimizer.m.clone(),
                hv=alg.hist_encoder_optimizer.v.clone(), steps=(alg.optimizer.step, alg.hist_encoder_optimizer.step), counter=alg.counter,
                gen=alg._rng().get_state(), storage_step=alg.storage.step)


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert (torch.equal(a[k], b[k]) if isinstance(a[k], torch.Tensor) else a[k] == b[k]), k


def test_round_trip_restores_parameters_adam_counter_and_generator(tmp_path):
    alg = make_alg()
    train_like(alg, 1)
    torch.save({"alg": alg.state_dict(), "iter": 5}, tmp_path / "ckpt.pt")
    saved = snapshot(alg)
    after_save = torch.randperm(40, generator=alg.generator)

    ck = torch.load(tmp_path / "ckpt.pt")                   # weights_only: the checkpoint is tensors, numbers and containers only
    fresh = make_alg(seed=3)
    fresh._packed = True
    fresh.storage.step = 2                                  # a live object in the middle of a rollout rolls back to the iteration boundary
    fresh.load_state_dict(ck["alg"])
    assert_same(snapshot(fresh), saved)
    assert fresh._packed is False                           # the tensor-core weight images are stale
    assert torch.equal(torch.randperm(40, generator=fresh.generator), after_save)
    assert fresh.get_value_mixing_ratio() == alg.get_value_mixing_ratio() and fresh.get_priv_reg_coef() == alg.get_priv_reg_coef()

    # a checkpoint taken before the first update (Adam step 0, empty optimizer state) clears the moments of the object it loads into
    zero = make_alg(seed=4)
    zero_sd = zero.state_dict()
    assert zero_sd["optimizer"]["state"] == {} and zero_sd["hist_encoder_optimizer"]["state"] == {}
    fresh.load_state_dict(zero_sd)
    assert_same(snapshot(fresh), snapshot(zero))


def test_default_generator_when_the_algorithm_has_none():
    """With `generator=None` act() and draw_indices() draw from the device's default generator: that is the state saved."""
    alg, other = make_alg(), make_alg(seed=2)
    alg.generator = other.generator = None
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(9)
        sd = alg.state_dict()
        expect = alg.storage.draw_indices(2)[0]
        torch.manual_seed(10)
        other.load_state_dict(sd)
        assert torch.equal(other.storage.draw_indices(2)[0], expect)


def test_save_in_the_middle_of_a_rollout_is_refused():
    alg = make_alg()
    alg.storage.step = 1
    with pytest.raises(L.DwbcError, match="between iterations"):
        alg.state_dict()


def refused(target, sd):
    before = snapshot(target)
    with pytest.raises(L.DwbcError):
        target.load_state_dict(sd)
    assert_same(snapshot(target), before)


@pytest.mark.parametrize("other", ["hist20", "hist50", "actor256", "envs8", "version", "hist_adam", "generator", "counter"])
def test_refused_load_changes_nothing(other):
    src = make_alg()
    train_like(src, 1)
    sd = src.state_dict()
    target = make_alg(seed=5)
    train_like(target, 6)
    if other == "hist20":                                   # same parameter names, other conv shapes
        sd = make_alg(num_hist=20).state_dict()
    elif other == "hist50":                                 # one more conv layer
        sd = make_alg(num_hist=50).state_dict()
    elif other == "actor256":
        sd = make_alg(actor_hidden_dims=(256,)).state_dict()
    elif other == "envs8":
        sd = make_alg(envs=8).state_dict()
    elif other == "version":
        sd["version"] = 2
    elif other == "hist_adam":                              # checked after the parameters and the main optimizer
        st = sd["hist_encoder_optimizer"]["state"]
        st[1]["exp_avg"] = st[1]["exp_avg"][:-1]
    elif other == "generator":                              # checked last: a CUDA Philox state does not fit a CPU generator
        sd["generator"] = torch.zeros(16, dtype=torch.uint8)
    elif other == "counter":
        sd["counter"] = -1
    refused(target, sd)
