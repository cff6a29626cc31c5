"""iPLAN-FC behaviour module on the CPU: the oracle (tools/beh_fc_oracle.py) pinned to the reference's own
nova/behavior_FC_policy module (tests/golden/behavior_learn_fc_{mpe,highway}.pt, written by
tests/golden/make_golden_fc.py), the termination-mask quirk, and the shape envelope of the two native entry points (each
rejection happens before the entry point's first CUDA call, so no device is needed and no pointer is followed)."""
import ctypes as C
import os
import re
import sys
from types import SimpleNamespace

import pytest
import torch

from tools.beh_fc_oracle import behavior_learn_fc_agent, fc_latent_update

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = C.c_void_p(0x1000)            # non-null, never dereferenced


def _case(golden_dir, case):
    if golden_dir not in sys.path:
        sys.path.insert(0, golden_dir)
    from beh_fc_inputs import load_fc_case
    return load_fc_case(golden_dir, case)


def _run_oracle(g, a, terminated=None, dtype=torch.float32):
    args = SimpleNamespace(**g["args"])
    d = g["data"]
    hist = d["history"][:, :-1, a].to(dtype)
    term = (d["terminated"] if terminated is None else terminated)[:, :-1, a, 0].to(dtype)
    ep = {k: v.clone().to(dtype) for k, v in g["enc_before"][a].items()}
    dp = {k: v.clone().to(dtype) for k, v in g["dec_before"][a].items()}
    out, _ = behavior_learn_fc_agent(ep, dp, hist, term, args)
    return out, ep, dp


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_fc_oracle_matches_reference(golden_dir, case):
    """One recorded ``learn`` call: per agent-net loss and post-step weights (within the fixture's float16 storage of the
    weight change), agent-net 0's clipped gradients 1e-6 relative per tensor; the logged sums and the return shape."""
    g = _case(golden_dir, case)
    args = SimpleNamespace(**g["args"])
    for a in range(args.n_agents):
        out, ep, dp = _run_oracle(g, a)
        assert abs(out["behavior_loss"] - g["behavior_loss"][a]) <= 1e-6 * abs(g["behavior_loss"][a])
        if a == 0:
            ref_g = g["grads0"]
            assert set(ref_g) == set(out["clipped"])
            for k in ref_g:
                rel = float((out["clipped"][k] - ref_g[k]).abs().max() / (ref_g[k].abs().max() + 1e-12))
                assert rel <= 1e-6, (k, rel)
        worst = max(max(float((ep[k] - g["enc_after"][a][k]).abs().max()) for k in ep),
                    max(float((dp[k] - g["dec_after"][a][k]).abs().max()) for k in dp))
        assert worst <= 1e-7, worst
    assert g["stability_loss"] == [] and g["total_loss"] == g["behavior_loss"]
    stats = g["stats"]
    key = [k for k in stats if k.endswith("behavior_loss")][0]
    assert abs(stats[key] - sum(g["behavior_loss"])) < 1e-5 * abs(stats[key])


def test_fc_oracle_termination_has_no_effect():
    """The reference's next-window mask stays all ones (:135-140): a batch that differs only in ``terminated`` gives the
    same loss and gradients.  Fixture-free: random weights and episode."""
    gen = torch.Generator().manual_seed(5)
    args = SimpleNamespace(max_history_len=4, latent_dim=3, max_grad_norm=10.0, lr_behavior=1e-4, optim_eps=1e-5)
    B, T, N, o, E, Dh = 2, 12, 3, 2, 32, 64
    K0 = 4 * o
    u = lambda *s: torch.rand(*s, generator=gen, dtype=torch.float64) * 2 - 1
    enc = {"linear_1.weight": u(E, K0), "linear_1.bias": u(E), "linear_2.weight": u(E, E), "linear_2.bias": u(E),
           "out.weight": u(3, E), "out.bias": u(3)}
    dec = {"decoder.linear_1.weight": u(Dh, K0 + 3), "decoder.linear_1.bias": u(Dh), "decoder.linear_2.weight": u(Dh, Dh),
           "decoder.linear_2.bias": u(Dh), "decoder.out.weight": u(K0, Dh), "decoder.out.bias": u(K0)}
    hist = u(B, T, N, o)
    outs = []
    for mask in (torch.zeros(B, T, dtype=torch.float64), (torch.rand(B, T, generator=gen) < 0.5).double()):
        ep = {k: v.clone() for k, v in enc.items()}
        dp = {k: v.clone() for k, v in dec.items()}
        outs.append(behavior_learn_fc_agent(ep, dp, hist, mask, args)[0])
    assert outs[0]["behavior_loss"] == outs[1]["behavior_loss"]
    assert all(torch.equal(outs[0]["grads"][k], outs[1]["grads"][k]) for k in outs[0]["grads"])


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_fc_oracle_latent_update_matches_reference(golden_dir, case):
    g = _case(golden_dir, case)
    for st in g["latent_steps"]:
        lat = fc_latent_update(g["enc_after"], st["window"])
        assert float((lat - st["latent"]).abs().max()) < 1e-6


def test_fc_oracle_rejects_episodes_without_a_position(golden_dir):
    g = _case(golden_dir, "mpe")
    args = SimpleNamespace(**g["args"])
    W = args.max_history_len
    hist = g["data"]["history"][:, :W + 1, 0]
    ep = {k: v.clone() for k, v in g["enc_before"][0].items()}
    dp = {k: v.clone() for k, v in g["dec_before"][0].items()}
    with pytest.raises(RuntimeError):
        behavior_learn_fc_agent(ep, dp, hist, torch.zeros(hist.shape[:2]), args)


# ---- native shape envelope ---------------------------------------------------------------------------------------------
def _lib():
    from iplan_b200 import _lib
    return _lib


def _rejects(rc, *needles):
    msg = _lib().lib.iplan_last_error().decode()
    assert rc != 0, f"accepted; last error {msg!r}"
    for n in needles:
        assert n in msg, (n, msg)


def _header_define(name):
    text = open(os.path.join(ROOT, "include", "iplan_b200.h")).read()
    return int(re.search(rf"#define {name} (\d+)", text).group(1))


def _view(dim):
    return _lib().View(0x1000, 64 * 64 * dim, 64 * dim, dim)


def _fc_step(obs_dim=5, latent_dim=8, hist_len=10, enc_hidden=32, win_stride=0, win_pad=0, n_slots=7):
    L = _lib()
    n0 = L.launch_count()
    rc = L.lib.iplan_behavior_fc_step(FAKE, 1024, _view(max(1, hist_len * obs_dim)), win_stride, win_pad, _view(max(1, latent_dim)),
                                      3, 2, n_slots, obs_dim, latent_dim, hist_len, enc_hidden, None)
    assert L.launch_count() == n0
    return rc


def _fc_learn(obs_dim=5, latent_dim=8, hist_len=10, n_steps=30, enc_hidden=32, dec_hidden=64):
    L = _lib()
    n0 = L.launch_count()
    rc = L.lib.iplan_beh_fc_learn(FAKE, 1024, FAKE, 4096, FAKE, FAKE, FAKE, 0.1, FAKE, 2, 3, n_steps, 7, obs_dim, latent_dim,
                                  hist_len, enc_hidden, dec_hidden, None)
    assert L.launch_count() == n0
    return rc


def test_fc_header_limits():
    assert _header_define("IPLAN_BFC_ENC_HIDDEN") == 32 and _header_define("IPLAN_BFC_DEC_HIDDEN") == 64
    assert _header_define("IPLAN_BFC_MAX_IN") == 64 and _header_define("IPLAN_BFC_MAX_LATENT") == 8


@pytest.mark.parametrize("entry", ["step", "learn"])
def test_fc_entry_points_reject_shapes_outside_their_limits(entry):
    call, tag = (_fc_step, "behavior_fc_step") if entry == "step" else (_fc_learn, "beh_fc_learn")
    _rejects(call(enc_hidden=31), tag, "enc_hidden 31 != 32")
    _rejects(call(enc_hidden=33), tag, "enc_hidden 33 != 32")
    _rejects(call(latent_dim=9, obs_dim=5, hist_len=10), tag, "latent_dim 9 not in [1,8]")
    _rejects(call(latent_dim=0), tag, "latent_dim 0 not in [1,8]")
    _rejects(call(obs_dim=0), tag, "obs_dim 0 < 1")
    _rejects(call(hist_len=0), tag, "hist_len 0 < 1")
    _rejects(call(obs_dim=5, hist_len=12, latent_dim=5), tag, "hist_len*obs_dim+latent_dim 65 > 64")
    _rejects(call(obs_dim=1, hist_len=57, latent_dim=8), tag, "hist_len*obs_dim+latent_dim 65 > 64")


def test_fc_step_rejects_window_padding_outside_the_window():
    _rejects(_fc_step(win_stride=100, win_pad=10), "behavior_fc_step", "win_pad 10 not in [0,10)")
    _rejects(_fc_step(win_stride=100, win_pad=-1), "behavior_fc_step", "win_pad -1 not in [0,10)")


def test_fc_learn_rejects_decoder_width_and_short_episodes():
    _rejects(_fc_learn(dec_hidden=63), "beh_fc_learn", "dec_hidden 63 != 64")
    _rejects(_fc_learn(dec_hidden=65), "beh_fc_learn", "dec_hidden 65 != 64")
    _rejects(_fc_learn(n_steps=11, hist_len=10), "beh_fc_learn", "n_pos = n_steps - 1 - hist_len = 0 < 1")
