"""CPU: the library surface of CUDA-graph replay without a GPU: the new entry points and the DwbcStepDevice mirror, that the existing
structs keep their layout, what a NULL or malformed device record does, the Adam bias-correction rows against the host arithmetic of the eager path, and which changes
make FusedPPO re-capture its update graphs."""
import ctypes as C
import os

import numpy as np
import pytest

from dwbc_b200 import _lib as L


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    return L.lib()


def test_exports_and_struct_mirrors(lib):
    for name in ("dwbc_adam_bias_correction", "dwbc_step_device_size", "dwbc_post_physics_step_device", "dwbc_ppo_minibatch_grad_sched",
                 "dwbc_clip_adam_step_table"):
        assert name in L.EXPORTS, name
    assert lib.dwbc_step_device_size() == C.sizeof(L.StepDevice) == 384
    # the curriculum block of the device record mirrors the one of DwbcStepArgs, field for field
    first, end = L.StepArgs.lin_vel_x.offset, L.StepArgs.generic_kernel.offset
    assert end - first == C.sizeof(L.StepDevice) - L.StepDevice.lin_vel_x.offset
    for name in ("ang_vel_yaw", "goal_l", "goal_p", "goal_y", "leg_scale", "arm_scale", "leg_termination_scale", "arm_termination_scale"):
        assert getattr(L.StepArgs, name).offset - first == getattr(L.StepDevice, name).offset - L.StepDevice.lin_vel_x.offset, name
    # the structs of ABI version 5 keep their layout: a caller built against the version-5 header stays right
    assert L.ABI_VERSION == 5
    assert [f for f, _ in L.StepArgs._fields_][-1] == "reserved_"
    assert [f for f, _ in L.PpoHyper._fields_][-1] == "arm_coefs"


def test_device_entry_points_refuse_null_records(lib):
    """The device-record entry points require their record; NULL is refused before anything is launched."""
    hp = L.PpoHyper()
    fake = 1 << 40
    assert lib.dwbc_clip_adam_step_table(fake, fake, fake, fake, 0, 16, C.addressof(hp), 1, None, fake, None, None) == -1
    assert lib.dwbc_ppo_minibatch_grad_sched(fake, fake, fake, fake, 16, C.addressof(hp), None, fake, fake, fake, None) == -1
    assert lib.dwbc_post_physics_step_device(None, None, None, fake, None) == -1


def test_bias_correction_rejects_bad_arguments(lib):
    hp = L.PpoHyper()
    hp.lr, hp.beta1, hp.beta2 = 1e-3, 0.9, 0.999
    out = (C.c_float * 4)()
    assert lib.dwbc_adam_bias_correction(None, 1, 2, out) == -1
    assert lib.dwbc_adam_bias_correction(C.addressof(hp), 0, 2, out) == -1
    assert lib.dwbc_adam_bias_correction(C.addressof(hp), 1, 2, None) == -1
    assert lib.dwbc_adam_bias_correction(C.addressof(hp), 1, 0, out) == 0


@pytest.mark.parametrize("lr,beta1,beta2", [(2e-4, 0.9, 0.999), (1e-3, 0.85, 0.995), (3.3e-5, 0.5, 0.9)])
def test_bias_correction_rows_are_the_host_floats(lr, beta1, beta2):
    """Row k of the table = what dwbc_clip_adam_step computes on the host for step first + k: the float32 hyper-parameters widened to
    double, 1 - beta^step with the C library's pow, then rounded to float32 (the same expression evaluated here through Python's pow)."""
    hp = L.PpoHyper()
    hp.lr, hp.beta1, hp.beta2 = lr, beta1, beta2
    first, n = 137, 60
    rows = L.adam_bias_correction(hp, first, n)
    f = lambda x: float(np.float32(x))  # noqa: E731
    for k in range(n):
        step = first + k
        bc1, bc2 = 1.0 - f(beta1) ** step, 1.0 - f(beta2) ** step
        assert rows[k, 0] == np.float32(f(lr) / bc1) and rows[k, 1] == np.float32(bc2 ** 0.5), k


def test_device_record_needs_the_tma_kernel(lib):
    """A device step record on a call that would take the warp-per-env kernel is refused before anything is launched."""
    import torch  # noqa: F401
    from dwbc_b200 import WidowGo1Params
    from dwbc_b200.env import make_env_cfg
    p = WidowGo1Params(num_envs=64)
    cfg = make_env_cfg(p, 64)
    buf = L.EnvBuffers()
    fake = 1 << 40
    for name, _ in L.EnvBuffers._fields_:
        if name not in ("obs_stride", "store_gamma", "reserved_", "store_values", "store_rewards", "store_dones", "height_samples",
                        "measured_heights", "heights_obs"):
            setattr(buf, name, fake)
    buf.obs_stride = p.num_obs
    args = L.StepArgs()
    args.generic_kernel = 1
    assert lib.dwbc_post_physics_step_device(C.addressof(cfg), C.addressof(buf), C.addressof(args), None, None) == -1
    assert lib.dwbc_post_physics_step_device(C.addressof(cfg), C.addressof(buf), C.addressof(args), fake, None) == -2


def _alg(N=16, T=4, **kw):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cpu", seed=0, num_priv=24, num_hist=10, num_prop=76)
    alg = FusedPPO(ac, device="cpu", num_mini_batches=2, num_learning_epochs=2, cuda_graphs=True, **kw)
    alg.init_storage(N, T, [860], [None], [18])
    if alg.torque_supervision:
        alg.set_arm_default_coeffs([20.0] * 6, [0.5] * 6, [0.1] * 6)
    alg._fill_hp()
    return alg


def test_graph_key(lib):
    alg = _alg()
    k0 = alg.graph_key("ppo")
    assert alg.graph_key("dagger") != k0
    alg.counter += 7                                      # schedules move: replayed with new device values, no re-capture
    alg._fill_hp()
    assert alg.graph_key("ppo") == k0
    alg.precision = "tf32"
    assert alg.graph_key("ppo") != k0
    alg.precision = "tf32x3"
    assert alg.graph_key("ppo") == k0
    alg.num_mini_batches = 4
    assert alg.graph_key("ppo") != k0
    alg.num_mini_batches = 2
    alg.init_storage(32, 4, [860], [None], [18])          # storage shape (and buffers, workspace) change
    assert alg.graph_key("ppo") != k0
    alg2 = _alg(torque_supervision=True)
    assert alg2.graph_key("ppo")[11] is True and k0[11] is False
    alg.clip_param = 0.3                                  # a by-value hyper-parameter of the captured launches
    alg._fill_hp()
    assert alg.graph_key("ppo")[12] != k0[12]


def test_multi_gpu_is_refused(lib):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cpu", seed=0, num_priv=24, num_hist=10, num_prop=76)
    with pytest.raises(L.DwbcError, match="all-reduce"):
        FusedPPO(ac, device="cpu", world_size=2, cuda_graphs=True)
