"""NumPy restatement of the library's in-kernel noise (iplan_b200/csrc/common.cuh: philox4x32, u01) and of the stream
layout of every kernel that draws from it.

Each kernel has two noise paths: explicit noise passed in by the caller (the parity tests), and Philox draws made inside
the kernel (training and the benchmark).  The functions below return exactly what the Philox path draws, in the layout
of that kernel's explicit-noise argument, so that a production call can be replayed into the float64 oracle.

Which Python counter feeds which consumer:
  * ``Prediction_policy.calls``: the K1 GAT step (``gat_step`` / ``GAT_latent_update``) and ``learn`` (pred_learn.cu)
    share it; every call advances it by one, except the pipelined ``GAT_latent_update`` (csrc/host_api.cu), where
    chunk c uses ``calls + c`` and the call advances it by the number of chunks;
  * ``DcntrlMAC.calls``: the sampling uniforms of K1c (controller_step.cu);
  * ``Behavior_policy.learn_calls`` (soft and hard module): the decoder dropout of the behaviour learner;
  * ``GAT128.calls``: the attention kernel of gat128.cu.
The seed of every module is ``args.seed`` (``GAT128``: 112358 + its constructor seed).
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al. 2011), as common.cuh:philox4x32.  ctr [..., 4], key [..., 2] (broadcast against each
    other), any integer dtype holding 32-bit words -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    shape = np.broadcast_shapes(ctr.shape[:-1], key.shape[:-1])
    x0, x1, x2, x3 = (np.broadcast_to(ctr[..., i], shape).copy() for i in range(4))
    k0, k1 = (np.broadcast_to(key[..., i], shape).copy() for i in range(2))
    for _ in range(10):
        p0 = _M0 * x0                                  # < 2^64: exact in uint64
        p1 = _M1 * x2
        x0, x1, x2, x3 = (p1 >> np.uint64(32)) ^ x1 ^ k0, p1 & _LO, (p0 >> np.uint64(32)) ^ x3 ^ k1, p0 & _LO
        k0 = (k0 + _W0) & _LO
        k1 = (k1 + _W1) & _LO
    return np.stack([x0, x1, x2, x3], axis=-1).astype(np.uint32)


def u01(bits):
    """common.cuh:u01, bit for bit: the top 24 bits plus one half (rounded to even in float32 from 2^23 up), times
    2^-24, capped at 1 - 2^-24, the largest float32 below 1.  The result lies in [2^-25, 1 - 2^-24], so neither log(u)
    nor log(1 - u) is infinite."""
    b = np.asarray(bits, dtype=np.uint32)
    u = ((b >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    return np.minimum(u, np.float32(1.0 - 2.0 ** -24))


def _words(lo_index, counter, key):
    """philox4x32((index lo, index hi, counter lo, counter hi), key) for an array of 64-bit indices -> uint32 [..., 4]."""
    idx = np.asarray(lo_index, dtype=np.uint64)
    c = np.uint64(counter)
    ctr = np.stack([idx & _LO, idx >> np.uint64(32), np.full_like(idx, c & _LO), np.full_like(idx, c >> np.uint64(32))], axis=-1)
    return philox4x32_10(ctr, np.asarray(key, dtype=np.uint64))


def draw_uniforms(draws, counter, key):
    """u01 of word (draw & 3) of Philox block (draw >> 2): every consumer below names its draws this way."""
    d = np.asarray(draws, dtype=np.uint64)
    w = _words(d >> np.uint64(2), counter, key)
    return u01(np.take_along_axis(w, (d & np.uint64(3)).astype(np.int64)[..., None], axis=-1)[..., 0])


def _seed_key(seed, xor_lo=0, xor_hi=0):
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return np.array([(s & 0xFFFFFFFF) ^ xor_lo, (s >> 32) ^ xor_hi], dtype=np.uint64)


def logistic_gumbel(u):
    """The two terms the kernels subtract, log(u) and log(1 - u), each rounded to float32, as a gumbel pair
    [..., 2] with [..., 1] - [..., 0] = log(u) - log(1 - u), the Logistic(0, 1) noise of one hard-attention edge.  (The
    kernels compute the logarithms in float32 — K1 and gat128 with the fast ``__logf`` — so the replay agrees with
    them to the accuracy of those logarithms, not bit for bit.)"""
    u = np.asarray(u, dtype=np.float64)
    return np.stack([np.log1p(-u), np.log(u)], axis=-1).astype(np.float32)


def _drop_self(x, N):
    """[..., N, N] over (ego i, slot j) -> [..., N, N-1] over (ego i, neighbour position s): s = j for j < i, j - 1 above."""
    keep = ~np.eye(N, dtype=bool)
    return x[..., keep].reshape(*x.shape[:-2], N, N - 1)


def gat_step_draws(n_agents, n_envs, n_slots):
    """K1 attention kernel (csrc/gat_step.cu:404-427): ego i of env b, agent-net ag, reads Philox block
    ((ag * n_envs + b) * N + i) * 16 + (j >> 2), key ``seed``, word j & 3 for slot j.  ``n_envs`` is the env count of the
    launch (chunk-local on the pipelined host path).  Draw ids [A, B, N, N-1] in neighbour order (s = j, or j - 1 past i)."""
    A, B, N = n_agents, n_envs, n_slots
    ego = np.arange(A * B * N, dtype=np.uint64).reshape(A, B, N, 1)
    return _drop_self(ego * np.uint64(64) + np.arange(N, dtype=np.uint64), N)


def gat_step_uniforms(seed, counter, n_agents, n_envs, n_slots, envs=None):
    """The uniforms of one K1 launch, [A, B, N, N-1]; ``envs``: only these envs of the launch, [A, len(envs), N, N-1]."""
    d = gat_step_draws(n_agents, n_envs, n_slots)
    return draw_uniforms(d if envs is None else d[:, list(envs)], counter, _seed_key(seed))


def gat_step_gumbel(seed, counter, n_agents, n_envs, n_slots, envs=None):
    """The noise of one K1 launch as ``gat_step``'s explicit ``gumbel`` argument: float32 [A, B, N, N-1, 2]."""
    return logistic_gumbel(gat_step_uniforms(seed, counter, n_agents, n_envs, n_slots, envs))


def gat_latent_update_gumbel(seed, calls0, n_agents, chunk_ends, n_slots):
    """The noise of one pipelined ``GAT_latent_update`` (csrc/host_api.cu:70-86): the envs are cut at ``chunk_ends``
    (``_lib.wave_chunks``), chunk c is a launch over its own envs with counter ``calls0 + c``.  [A, B, N, N-1, 2]."""
    parts, lo = [], 0
    for c, hi in enumerate(chunk_ends):
        if hi > lo:
            parts.append(gat_step_gumbel(seed, calls0 + c, n_agents, hi - lo, n_slots))
        lo = hi
    return np.concatenate(parts, axis=1)


def gat128_draws(n_agents, n_items, n_slots=16):
    """gat128 attention kernel (csrc/gat128.cu:284-293): edge ((ag * items + item) * 16 + i) * 15 + s is the Philox block,
    key ``seed``, word 0.  Draw ids [A, items, 16, 15]."""
    e = np.arange(n_agents * n_items * n_slots * (n_slots - 1), dtype=np.uint64) * np.uint64(4)
    return e.reshape(n_agents, n_items, n_slots, n_slots - 1)


def gat128_gumbel(seed, counter, n_agents, n_items, n_slots=16):
    """``GAT128.forward``'s explicit ``gumbel``: [A, items, 16, 15, 2]."""
    return logistic_gumbel(draw_uniforms(gat128_draws(n_agents, n_items, n_slots), counter, _seed_key(seed)))


def controller_draws(n_agents, n_envs):
    """K1c sampling (csrc/controller_step.cu:446-449): row ob = ag * n_envs + b is the Philox block, key
    (seed lo, seed hi ^ 0x5bd1e995), word 0.  Draw ids [A, B]."""
    return (np.arange(n_agents * n_envs, dtype=np.uint64) * np.uint64(4)).reshape(n_agents, n_envs)


def controller_uniforms(seed, counter, n_agents, n_envs):
    """K1c's ``uniforms`` argument: float32 [A, B]."""
    return draw_uniforms(controller_draws(n_agents, n_envs), counter, _seed_key(seed, xor_hi=0x5BD1E995))


def pred_learn_draws(n_agents, P, n_slots, pred_length, hid=32):
    """pred_learn.cu, sample = ag * P + p: the Gumbel draw of ego i, neighbour s is Philox block
    (sample * N + i) * (N-1) + s, key ``seed``, word 0 (:206-213); the dropout draw of decoder step t, node n, unit c is
    block ((sample * pl + t) * N + n) * 32 + c, key (seed lo ^ 0x9e3779b9, seed hi), word 0 (:268-274).
    Draw ids ([A, P, N, N-1], [A, P, pl, N, 32])."""
    A, N = n_agents, n_slots
    g = np.arange(A * P * N * (N - 1), dtype=np.uint64).reshape(A, P, N, N - 1) * np.uint64(4)
    k = np.arange(A * P * pred_length * N * hid, dtype=np.uint64).reshape(A, P, pred_length, N, hid) * np.uint64(4)
    return g, k


def pred_learn_noise(seed, counter, n_agents, P, n_slots, pred_length, p_drop, hid=32):
    """``debug_learn``'s (gumbel float32 [A, P, N, N-1, 2], keep uint8 [A, P, pl, N, 32]) of one ``learn`` call: an
    element is kept when its u01 >= p_drop."""
    g, k = pred_learn_draws(n_agents, P, n_slots, pred_length, hid)
    ug = draw_uniforms(g, counter, _seed_key(seed))
    uk = draw_uniforms(k, counter, _seed_key(seed, xor_lo=0x9E3779B9))
    return logistic_gumbel(ug), (uk >= np.float32(p_drop)).astype(np.uint8)


def beh_learn_draws(n_agents, n_envs, n_pos, n_slots, hist_len, hid=64):
    """beh_learn_tile.cu:583-597 (every window geometry: soft n_pos = T - 1 - W, hard n_pos = T / W - 1): chain
    gid = (ag * B + b) * N + n reads Philox block e = ((gid * n_pos + j) * W + w) * 16 + ug, key
    (seed lo ^ 0x85ebca6b, seed hi); word i is unit ug + 16 i.  Draw ids [A, B, n_pos, N, W, 64] (``debug_keep``'s layout)."""
    A, B, N, W, G = n_agents, n_envs, n_slots, hist_len, hid // 4
    e = np.arange(A * B * N * n_pos * W * G, dtype=np.uint64).reshape(A, B, N, n_pos, W, 1, G) * np.uint64(4)
    d = e + np.arange(4, dtype=np.uint64).reshape(4, 1)                  # [A, B, N, n_pos, W, i, ug]: unit 16 i + ug
    return d.reshape(A, B, N, n_pos, W, hid).transpose(0, 1, 3, 2, 4, 5)


def beh_learn_keep(seed, counter, n_agents, n_envs, n_pos, n_slots, hist_len, p_drop, hid=64):
    """``debug_keep`` of one behaviour ``learn`` call: uint8 [A, B, n_pos, N, W, 64], kept when u01 >= p_drop.  Each
    Philox block is computed once for its four words; ``beh_learn_draws`` names the same draws one by one."""
    A, B, N, W = n_agents, n_envs, n_slots, hist_len
    key = _seed_key(seed, xor_lo=0x85EBCA6B)
    per = B * N * n_pos * W * (hid // 4)
    out = []
    for ag in range(A):                                                   # one agent-net at a time: bounded memory
        e = np.arange(ag * per, (ag + 1) * per, dtype=np.uint64)
        k = u01(_words(e, counter, key)) >= np.float32(p_drop)          # [(b, n, j, w, ug), i]
        k = k.reshape(B, N, n_pos, W, hid // 4, 4).transpose(0, 2, 1, 3, 5, 4).reshape(B, n_pos, N, W, hid)
        out.append(k.astype(np.uint8))
    return np.stack(out)
