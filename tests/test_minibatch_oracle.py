"""The mini-batch oracle (oracle/minibatch_oracle.py) against the reference's own IPPOLearner run with
num_mini_batch = 3 (tests/golden/learner_minibatch.pt, written by tests/golden/make_golden_minibatch.py), and the
host-side pieces of the mini-batch update that need no device.  CPU only."""
import os
from types import SimpleNamespace

import torch

from iplan_b200 import parallel
from oracle import iplan_oracle as O
from oracle import minibatch_oracle as M

STAT_KEYS = ("value_loss", "policy_loss", "dist_entropy", "actor_grad_norm", "critic_grad_norm", "ratio")


def _golden(golden_dir):
    from tests.golden.minibatch_fixture import load
    return load(os.path.join(golden_dir, "learner_minibatch.pt"))


def test_oracle_matches_reference_with_three_mini_batches(golden_dir):
    g = _golden(golden_dir)
    args = SimpleNamespace(**g["args"])
    k, n = args.num_mini_batch, args.batch_size * args.episode_limit
    assert k == 3 and n % k != 0
    all_stats = []
    for a in range(args.n_agents):
        ap = {key: v.clone() for key, v in g["actors_before"][a].items()}
        cp = {key: v.clone() for key, v in g["critics_before"][a].items()}
        stats, opt_a, opt_c = M.train_agent(ap, cp, M.agent_batch(g["data"], a, args.n_actions), a, args, g["perms"][a], k)
        for key in O.ACTOR_TRAINABLE:
            assert float((ap[key] - g["actors_after"][a][key]).abs().max()) < 1e-5, (a, key)
        for key in O.CRITIC_TRAINABLE:
            assert float((cp[key] - g["critics_after"][a][key]).abs().max()) < 1e-5, (a, key)
        assert opt_a.t == opt_c.t == g["opt_step"] == args.ppo_epoch * k
        all_stats += stats
    assert len(all_stats) == args.ppo_epoch * k * args.n_agents
    for key in STAT_KEYS:
        mine = sum(s[key] for s in all_stats) / len(all_stats)
        ref = [v for name, v in g["stats"].items() if name.endswith(key)][0]
        assert abs(mine - ref) < 1e-5 * max(1.0, abs(ref)), (key, mine, ref)


def test_sets_drop_the_trailing_rows_and_partition_the_rest(golden_dir):
    g = _golden(golden_dir)
    args = SimpleNamespace(**g["args"])
    n, k = args.batch_size * args.episode_limit, args.num_mini_batch
    perm = g["perms"][0, 0]
    sets = M.mini_batch_sets(perm, k)
    assert [len(s) for s in sets] == [n // k] * k
    assert torch.equal(torch.cat(sets), perm[:k * (n // k)])
    idx, count = parallel.local_minibatch_rows(g["perms"], k, args.episode_limit, 0, args.batch_size)
    assert tuple(idx.shape) == (args.n_agents, args.ppo_epoch, k, n // k) and bool((count == n // k).all())
    assert torch.equal(idx[0, 0], torch.stack(sets))


def test_all_dead_set_gives_finite_weights(golden_dir):
    """A set without an alive row: the policy and value terms are skipped, the weights stay finite and the critic,
    which has no other term, does not move."""
    g = _golden(golden_dir)
    args = SimpleNamespace(**dict(g["args"], ppo_epoch=1))
    data = {key: v.clone() for key, v in g["data"].items()}
    T, k = args.episode_limit, 7                      # sets of 7 rows; the identity permutation makes set 0 = episode 0
    data["terminated"][0, :, 0] = 1
    ap = {key: v.double() for key, v in g["actors_before"][0].items()}
    cp = {key: v.double() for key, v in g["critics_before"][0].items()}
    cp0 = {key: v.clone() for key, v in cp.items()}
    perm = torch.arange(args.batch_size * T)
    flat = M.agent_rows(ap, cp, M.agent_batch(data, 0, args.n_actions, torch.float64), 0, args)
    assert float(flat["alive"][perm[:T]].sum()) == 0.0
    e = M.ppo_set(ap, cp, flat, args, perm[:T])
    assert float(e["policy_loss"]) == 0.0 and float(e["value_loss"]) == 0.0
    assert all(float(v.abs().max()) == 0.0 for v in e["grads_critic"].values())
    stats, _, _ = M.train_agent(ap, cp, M.agent_batch(data, 0, args.n_actions, torch.float64), 0, args, [perm], k)
    assert len(stats) == k and all(torch.isfinite(torch.tensor([s[key] for key in STAT_KEYS])).all() for s in stats)
    assert all(bool(torch.isfinite(v).all()) for v in list(ap.values()) + list(cp.values()))
    assert any(not torch.equal(cp[key], cp0[key]) for key in O.CRITIC_TRAINABLE)     # the later sets did train it
