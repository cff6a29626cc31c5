"""oracle/philox.py, the NumPy restatement of the kernels' Philox noise: known answers of the generator, the range of the
bits-to-uniform map, and the statistics of every consumer's replayed stream at the benchmark's shape (Highway: 5
agent-nets, 55 slots, 512 envs).  The GPU side — that the kernels draw exactly these streams — is
tests/test_gpu_noise_streams.py."""
import math

import numpy as np
import pytest

from oracle import philox as PX

A, N, B = 5, 55, 512


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    """The Random123 known-answer vectors of Philox4x32-10."""
    got = PX.philox4x32_10(np.array(ctr), np.array(key))
    assert got.dtype == np.uint32 and tuple(int(x) for x in got) == want


def test_philox_vectorises_like_scalar_calls():
    rng = np.random.default_rng(0)
    ctr = rng.integers(0, 2 ** 32, size=(7, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, size=(7, 2), dtype=np.uint64)
    many = PX.philox4x32_10(ctr, key)
    for r in range(7):
        assert np.array_equal(many[r], PX.philox4x32_10(ctr[r], key[r]))


def test_u01_is_strictly_inside_the_unit_interval():
    """Every one of the 2^24 values of the top 24 bits (the low 8 bits are never read) maps strictly inside (0, 1), so
    log(u) and log(1 - u) are finite for every draw; the map is monotone.  Only the topmost input, whose float32 sum
    rounds to 2^24 (u = 1.0), differs from the uncapped map, so the cap leaves every other draw of every stream as it was."""
    x = np.arange(2 ** 24, dtype=np.uint32) << np.uint32(8)
    u = PX.u01(x)
    assert u.dtype == np.float32
    assert float(u.min()) > 0.0 and float(u.max()) < 1.0
    assert float(u.min()) == 2.0 ** -25 and float(u.max()) == 1.0 - 2.0 ** -24
    assert np.all(np.diff(u) >= 0)
    uncapped = ((x >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    assert float(uncapped[-1]) == 1.0
    assert np.array_equal(u[:-1], uncapped[:-1])
    g = PX.logistic_gumbel(u[[0, -1]])
    assert np.isfinite(g).all()
    low = PX.u01(np.arange(256, dtype=np.uint32))                     # bits below the 24 read ones do not matter
    assert np.all(low == low[0])


def _unique(ids):
    ids = np.asarray(ids).reshape(-1)
    return np.unique(ids).size == ids.size


def test_every_consumer_names_each_draw_once_per_call():
    """Within one call no two elements of a consumer read the same Philox word (a wrong stride or word index would
    share noise between agent-nets, envs, egos or units)."""
    assert _unique(PX.gat_step_draws(A, B, N))
    assert _unique(PX.gat128_draws(32, 64))
    assert _unique(PX.controller_draws(A, B))
    g, k = PX.pred_learn_draws(A, 64, N, 5)
    assert _unique(g) and _unique(k)
    soft = PX.beh_learn_draws(A, 8, 90 - 1 - 10, N, 10)             # soft window geometry, T = 90, W = 10
    hard = PX.beh_learn_draws(A, 8, 90 // 10 - 1, N, 10)            # hard window geometry
    assert _unique(soft) and _unique(hard)
    assert soft.shape == (A, 8, 79, N, 10, 64) and hard.shape == (A, 8, 8, N, 10, 64)


def test_beh_learn_keep_blockwise_equals_drawwise():
    """beh_learn_keep computes each Philox block once for its four units; it must agree with naming the draws one by one."""
    d = PX.beh_learn_draws(2, 3, 4, 5, 6)
    u = PX.draw_uniforms(d, 9, PX._seed_key(77, xor_lo=0x85EBCA6B))
    assert np.array_equal(PX.beh_learn_keep(77, 9, 2, 3, 4, 5, 6, 0.1), (u >= np.float32(0.1)).astype(np.uint8))


def _within_5_sigma(x, p):
    return abs(float(x.mean()) - p) < 5 * math.sqrt(p * (1 - p) / x.size)


def test_dropout_keep_rate():
    """Keep rate 0.9 within 5 sigma for both learners' dropout streams."""
    _, keep = PX.pred_learn_noise(112358, 3, A, 64, N, 5, 0.1)
    assert _within_5_sigma(keep, 0.9)
    keep = PX.beh_learn_keep(112358, 0, 2, 4, 79, N, 10, 0.1)
    assert _within_5_sigma(keep, 0.9)


def test_logistic_noise_moments():
    """K1's noise at the benchmark shape: Logistic(0, 1), mean 0 and variance pi^2 / 3 (kurtosis makes the variance's
    standard error about 2.2 times that of a Gaussian)."""
    g = PX.gat_step_gumbel(112358, 0, A, B, N)
    noise = (g[..., 1].astype(np.float64) - g[..., 0])
    n = noise.size
    var = math.pi ** 2 / 3
    assert abs(noise.mean()) < 5 * math.sqrt(var / n)
    assert abs(noise.var() - var) < 5 * var * math.sqrt(3.2 / n)


def test_streams_are_uncorrelated_across_agent_nets_and_calls():
    """Correlation near 0 between the agent-nets of one K1 launch and between consecutive calls (counter c, c + 1) of K1,
    K1c and the behaviour learner's dropout."""
    u = PX.gat_step_uniforms(112358, 4, A, 64, N).reshape(A, -1).astype(np.float64)
    bound = 5 / math.sqrt(u.shape[1])
    c = np.corrcoef(u)
    assert np.abs(c[~np.eye(A, dtype=bool)]).max() < bound
    for stream in (lambda k: PX.gat_step_uniforms(112358, k, A, 64, N),
                   lambda k: PX.controller_uniforms(112358, k, A, 4096),
                   lambda k: PX.beh_learn_keep(112358, k, 1, 2, 20, N, 10, 0.1)):
        x, y = (stream(k).reshape(-1).astype(np.float64) for k in (6, 7))
        assert abs(np.corrcoef(x, y)[0, 1]) < 5 / math.sqrt(x.size)


def test_pipelined_chunks_use_their_own_counter_and_env_range():
    """The pipelined GAT_latent_update's noise is chunk c's own launch (chunk-local envs, counter calls0 + c): distinct
    chunks, and so distinct counters, never repeat a uniform block."""
    ends = [40, 80, 130]
    g = PX.gat_latent_update_gumbel(112358, 10, A, ends, N)
    assert g.shape == (A, 130, N, N - 1, 2)
    assert np.array_equal(g[:, 40:80], PX.gat_step_gumbel(112358, 11, A, 40, N))
    assert np.array_equal(g[:, 80:], PX.gat_step_gumbel(112358, 12, A, 50, N))
    assert not np.array_equal(g[:, :40], g[:, 40:80])
