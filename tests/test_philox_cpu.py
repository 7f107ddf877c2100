"""CPU: a numpy restatement of the env's random stream -- Philox4x32-10 (Salmon et al., SC'11) and the 24-bit uniform `u01` of
csrc/common.cuh -- pinned to Random123's known-answer vectors.  tests/test_gpu_philox.py holds dwbc_fill_uniform to this restatement bit
for bit, and test_gpu_env.py's test_philox_mode_equals_table_mode holds the in-kernel draws to dwbc_fill_uniform, so the stream the
post-physics kernel draws is tied to the published algorithm rather than only to itself."""
import numpy as np
import pytest

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)          # round multipliers
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)          # Weyl key increments
LO32 = np.uint64(0xFFFFFFFF)
RAND_COLS = 104                                                 # columns of the env's uniform table (config.RAND_COLS)


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (c0, c1, c2, c3), key: two uint32 arrays (k0, k1), all broadcastable.  Returns the four uint32 output
    words.  Each round: (hi, lo) = 64-bit products M0 * c0 and M1 * c2; c = (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0); then the key
    is bumped by the Weyl increments."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint32) for k in key)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & LO32).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & LO32).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = k0 + W0, k1 + W1
    return c0, c1, c2, c3


def u01(x):
    """(x >> 8) * 2^-24: a float32 in [0, 1) on the 24-bit grid (exact in float32)."""
    return ((np.asarray(x, dtype=np.uint32) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def uniform_table(num_envs, seed, step):
    """What dwbc_fill_uniform writes: [num_envs, RAND_COLS] float32, column c of env e = u01 of word c % 4 of
    philox(ctr = (e, c // 4, step_lo, step_hi), key = (seed_lo, seed_hi)).  seed and step are unsigned 64-bit."""
    env = np.arange(num_envs, dtype=np.uint32)[:, None]
    block = np.arange(RAND_COLS // 4, dtype=np.uint32)[None, :]
    step, seed = int(step), int(seed)
    words = philox4x32_10((env, block, np.uint32(step & 0xFFFFFFFF), np.uint32(step >> 32)),
                          (np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32)))
    return u01(np.stack(words, axis=-1).reshape(num_envs, RAND_COLS))


# Random123 (kat_vectors, philox4x32 10 rounds): counter, key -> output
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,out", KAT, ids=["zeros", "ones", "pi"])
def test_restatement_gives_random123_known_answers(ctr, key, out):
    assert tuple(int(w) for w in philox4x32_10(ctr, key)) == out


def test_restatement_is_elementwise():
    """The array form computes each lane as the scalar form does (so the table below is the known-answer function, lane by lane)."""
    ctr = [np.array([c[i] for c, _, _ in KAT], dtype=np.uint32) for i in range(4)]
    key = [np.array([k[i] for _, k, _ in KAT], dtype=np.uint32) for i in range(2)]
    got = np.stack(philox4x32_10(ctr, key), axis=1)
    assert [tuple(int(w) for w in row) for row in got] == [o for _, _, o in KAT]


def test_u01_is_the_24_bit_grid():
    x = np.array([0, 0xFF, 0x100, 0x80000000, 0xFFFFFFFF], dtype=np.uint32)
    assert u01(x).tolist() == [0.0, 0.0, 2.0 ** -24, 0.5, 1.0 - 2.0 ** -24]


def test_table_layout():
    """Column c is word c % 4 of block c // 4; the step's high word and the seed's high word reach the counter and the key."""
    tab = uniform_table(3, 5, 7)
    assert tab.shape == (3, RAND_COLS) and tab.dtype == np.float32
    w = philox4x32_10((2, 9, 7, 0), (5, 0))
    assert tab[2, 36:40].tolist() == u01(np.array(w)).tolist()
    assert not np.array_equal(uniform_table(3, 5, 7 + (1 << 32)), tab)
    assert not np.array_equal(uniform_table(3, 5 + (1 << 32), 7), tab)
