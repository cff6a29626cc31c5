"""Pin the hard-update behaviour oracle (tools/beh_hard_oracle.py) to the reference's own nova/behavior_policy module
(tests/golden/behavior_learn_hard_{mpe,highway}.pt, written by tests/golden/make_golden_hard.py).  CPU only."""
import sys
from types import SimpleNamespace

import pytest
import torch

from oracle import iplan_oracle as O
from tools.beh_hard_oracle import behavior_learn_hard_agent


def _case(golden_dir, case):
    if golden_dir not in sys.path:
        sys.path.insert(0, golden_dir)
    from beh_hard_inputs import load_hard_case
    return load_hard_case(golden_dir, case)


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_behavior_learn_hard_matches_reference(golden_dir, case):
    """One recorded ``learn`` call with its dropout replayed: loss and post-step weights per agent-net, and the gradients
    as clipped by the reference for agent-net 0."""
    g = _case(golden_dir, case)
    args = SimpleNamespace(**g["args"])
    d = g["data"]
    hist = d["history"][:, :-1]
    term = d["terminated"][:, :-1, :, 0].float()
    for a in range(args.n_agents):
        mask = 1 - term[:, :, a] if args.env == "MPE" else term[:, :, a]
        ep = {k: v.clone() for k, v in g["enc_before"][a].items()}
        dp = {k: v.clone() for k, v in g["dec_before"][a].items()}
        out, _ = behavior_learn_hard_agent(ep, dp, hist[:, :, a], mask, g["dropout_keep"][a], args)
        assert abs(out["behavior_loss"] - g["behavior_loss"][a]) <= 1e-6 * abs(g["behavior_loss"][a])
        rel = 0.0
        if a == 0:
            ref_g = g["grads0"]
            assert set(ref_g) == set(out["clipped"])
            rel = max(float((out["clipped"][k] - ref_g[k]).abs().max() / (ref_g[k].abs().max() + 1e-12)) for k in ref_g)
        worst = max(max(float((ep[k] - g["enc_after"][a][k]).abs().max()) for k in ep),
                    max(float((dp[k] - g["dec_after"][a][k]).abs().max()) for k in dp))
        print(f"[behavior.learn hard {case} a={a}] loss {out['behavior_loss']:.6f} (reference {g['behavior_loss'][a]:.6f}); "
              + (f"worst relative gradient difference {rel:.2e}; " if a == 0 else "")
              + f"max |param - reference| after the step {worst:.2e}")
        assert rel <= 1e-6 and worst <= 1e-6
    stats = g["stats"]
    key = [k for k in stats if k.endswith("behavior_loss")][0]
    assert abs(stats[key] - sum(g["behavior_loss"])) < 1e-5 * abs(stats[key])


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_hard_mask_lag_changes_the_loss(golden_dir, case):
    """The fixture exercises the reference's one-window mask lag: weighting each target row by the mask at that row
    instead would give a different loss."""
    g = _case(golden_dir, case)
    args = SimpleNamespace(**g["args"])
    W = args.max_history_len
    d = g["data"]
    hist = d["history"][:, :-1]
    term = d["terminated"][:, :-1, :, 0].float()
    changed = 0
    for a in range(args.n_agents):
        mask = 1 - term[:, :, a] if args.env == "MPE" else term[:, :, a]
        unlagged = torch.cat([mask[:, W:], torch.zeros_like(mask[:, :W])], dim=1)
        ep = {k: v.clone() for k, v in g["enc_before"][a].items()}
        dp = {k: v.clone() for k, v in g["dec_before"][a].items()}
        out, _ = behavior_learn_hard_agent(ep, dp, hist[:, :, a], unlagged, g["dropout_keep"][a], args)
        changed += abs(out["behavior_loss"] - g["behavior_loss"][a]) > 1e-4 * abs(g["behavior_loss"][a])
    assert changed >= 1


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_hard_latent_update_is_the_soft_update_with_coefficient_one(golden_dir, case):
    """Three recorded ``latent_update`` calls of the reference's hard module (prev_latent ignored, hidden carried) against
    the soft-update oracle with coefficient 1 and the trained encoder."""
    g = _case(golden_dir, case)
    enc = g["enc_after"]
    for st in g["latent_steps"]:
        lat, hid = O.behavior_latent_update(enc, st["window"], st["hid_in"], st["prev"], coef=1.0)
        assert float((lat - st["latent"]).abs().max()) < 2e-6
        assert float((hid - st["hid_out"]).abs().max()) < 2e-6


def test_hard_oracle_rejects_partial_windows(golden_dir):
    g = _case(golden_dir, "mpe")
    args = SimpleNamespace(**g["args"])
    hist = g["data"]["history"][:, :-1, :, 0]
    mask = torch.ones(hist.shape[:2])
    ep = {k: v.clone() for k, v in g["enc_before"][0].items()}
    dp = {k: v.clone() for k, v in g["dec_before"][0].items()}
    with pytest.raises(RuntimeError):
        behavior_learn_hard_agent(ep, dp, hist[:, :25], mask[:, :25], g["dropout_keep"][0], args)
    with pytest.raises(RuntimeError):
        behavior_learn_hard_agent(ep, dp, hist[:, :10], mask[:, :10], g["dropout_keep"][0], args)
