"""GPU: dwbc_fill_uniform -- the uniform table of the in-kernel Philox stream, which test_gpu_env.py's test_philox_mode_equals_table_mode
ties to the post-physics kernel's own draws -- equals the numpy restatement of test_philox_cpu.py (pinned there to Random123's
known-answer vectors) bit for bit: every one of the 104 columns (block col // 4, word col % 4), seeds and steps at and above 2^32, the
step 2^32 - 1 whose successor carries into the counter's high word, more than 65536 envs, and the per-rank seeds of shard.rank_seed."""
import numpy as np
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import shard
from test_philox_cpu import RAND_COLS, uniform_table

pytestmark = pytest.mark.gpu


def fill_uniform(num_envs, seed, step):
    out = torch.empty(num_envs, RAND_COLS, device="cuda")
    L.check(L.lib().dwbc_fill_uniform(L.ptr(out), num_envs, seed, step, L.stream_ptr()), "dwbc_fill_uniform")
    return out.cpu().numpy()


def assert_bitwise(got, want, what):
    diff = got.view(np.uint32) != want.view(np.uint32)
    assert not diff.any(), f"{what}: {int(diff.sum())} of {diff.size} entries differ, first at {np.argwhere(diff)[0].tolist()}"


CASES = [(70001, 1, 150),                              # more than 65536 envs
         (1000, 5, (1 << 32) - 1), (1000, 5, 1 << 32),   # the last step of the low word, the first with a high word
         (1000, (1 << 32) + 3, 151),                     # a seed with a high word
         (1000, (1 << 40) + 17, (1 << 33) + 9),
         (37, (1 << 64) - 1, (1 << 64) - 1),
         (1, 0, 0)]


@pytest.mark.parametrize("N,seed,step", CASES)
def test_fill_uniform_equals_the_restatement(N, seed, step):
    got = fill_uniform(N, seed, step)
    assert_bitwise(got, uniform_table(N, seed, step), f"N={N} seed={seed} step={step}")
    assert got.min() >= 0.0 and got.max() < 1.0


def test_per_rank_seeds_draw_different_streams():
    """The seeds shard.rank_seed gives eight ranks differ, and each rank's table is the restatement's for its own seed."""
    N, step = 512, 150
    seeds = [shard.rank_seed(1000, r) for r in range(8)]
    assert len(set(seeds)) == 8
    tabs = []
    for s in seeds:
        tabs.append(fill_uniform(N, s, step))
        assert_bitwise(tabs[-1], uniform_table(N, s, step), f"rank seed {s}")
    for i in range(8):
        for j in range(i):
            assert float(np.mean(tabs[i] == tabs[j])) < 1e-3, (i, j)
