"""Inputs and output digests of the whole-episode observation-wrapper check: shared by make_golden.py, which records the
reference wrapper's outputs, and tests/test_gpu_rollout.py, which compares the package's wrapper with them."""
import hashlib

import numpy as np


def obs_episode_inputs(rng, B, A, N, M, o, L):
    """L + 1 timesteps of raw observations [B][A][M][o + 1] in which vehicles enter, leave and re-enter the agents' view, then
    the episode mask [B][L][A]; deterministic in `rng`."""
    pool = np.arange(1000, 1000 + N - 1)                # <= N - 1 other vehicles ever: the table never overflows
    steps = []
    for t in range(L + 1):
        obs = np.zeros((B, A, M, o + 1))
        for k in range(B):
            for i in range(A):
                n_seen = rng.integers(2, M + 1)
                hi = min(len(pool), 8 + t)              # the set an agent may meet grows; earlier ones drop out and return
                seen = rng.choice(pool[:hi], size=min(n_seen - 1, hi), replace=False)
                obs[k, i, 0, 0] = 7 + i
                obs[k, i, 0, 1:] = rng.uniform(-1, 1, size=o)
                obs[k, i, 1:1 + len(seen), 0] = seen
                obs[k, i, 1:1 + len(seen), 1:] = rng.uniform(-1, 1, size=(len(seen), o))
        steps.append(obs.astype(np.float32).astype(np.float64))     # both sides see fp32-representable values
    mask = (rng.uniform(size=(B, L, A)) < 0.8).astype(np.float64)
    return steps, mask


def f32_digest(x):
    """sha256 of an array's float32 bytes (C order) with its shape: equal digests = bit-equal float32 arrays."""
    a = np.ascontiguousarray(np.asarray(x, dtype=np.float32))
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()

