#!/usr/bin/env python
"""Golden fixture of the IPPO update with num_mini_batch > 1, recorded by RUNNING THE REFERENCE's own IPPOLearner on
the CPU (as make_golden.py does for num_mini_batch = 1; same helpers, needs the reference checkout it names).

A small MPE case (one agent, one landmark: N = 2 slots, F = 94), 8 episodes of T = 7, batch_size 7, num_mini_batch 3,
2 epochs: n = 49 rows per permutation, sets of 16, so that one trailing row per epoch is not trained on.  Saved:
inputs, weights before and after, the permutations generate_data drew (seeded th.randperm, agent-major then epoch), the
six logged statistics and the optimisers' step count.  minibatch_fixture.py describes how the weights are stored
(float16-exact initial weights; the update of the trained tensors as int16 steps of 2^-23) and reads the file back.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_minibatch.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import NullLogger, make_scheme, ref_args, sd_clone, synth_history  # noqa: E402
from minibatch_fixture import encode_after  # noqa: E402
from oracle.iplan_oracle import ACTOR_TRAINABLE, CRITIC_TRAINABLE  # noqa: E402


def small(sd):
    """float16 where it holds the values exactly."""
    return {k: v.half() if v.is_floating_point() and torch.equal(v.half().float(), v) else v for k, v in sd.items()}


def trained(after, before, keys):
    """The update of the trained tensors, encoded; every other entry must not have moved."""
    for k, v in after.items():
        assert k in keys or torch.equal(v, before[k]), k
    return encode_after(after, before, keys)


def main():
    from controllers.dcntrl_controller import DcntrlMAC
    from learners.ippo_learner import IPPOLearner
    from components.episode_buffer import EpisodeBatch

    args = ref_args("MPE", num_agents=1, num_landmarks=1, episode_length=7, buffer_size=8, batch_size=7, batch_size_run=8,
                    ppo_epoch=2, num_mini_batch=3)
    A, N, o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
    L, D, R, T, B = args.latent_dim, args.attention_dim, args.rnn_hidden_dim, args.episode_limit, args.batch_size_run
    assert T == 7 and (args.batch_size * T) % args.num_mini_batch != 0
    torch.manual_seed(4242)
    scheme, groups, preprocess = make_scheme(args)
    batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
    mac = DcntrlMAC(batch.scheme, groups, args)
    logger = NullLogger()
    learner = IPPOLearner(mac, batch.scheme, logger, args)
    with torch.no_grad():
        for ag in mac.agents:
            ag.act.action_out.linear.weight.mul_(30.0)
            ag.base.feature_norm.weight.uniform_(0.5, 1.5)
            ag.base.feature_norm.bias.uniform_(-0.2, 0.2)
        for cr in mac.critics:
            cr.base.feature_norm.weight.uniform_(0.5, 1.5)
            cr.base.feature_norm.bias.uniform_(-0.2, 0.2)
        for net in list(mac.agents) + list(mac.critics):
            for p in net.parameters():
                p.copy_(p.half().float())
    rng = np.random.default_rng(91)
    data = dict(
        history=np.stack([synth_history(rng, B, A, N, o, min(N, 3 + t)) for t in range(T + 1)], axis=1),
        attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
        behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
        rnn_states_actors=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
        rnn_states_critics=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
        actions=rng.integers(0, args.n_actions, size=(B, T + 1, A, 1)),
        avail_actions=np.ones((B, T + 1, A, args.n_actions), dtype=np.int64),
        reward=rng.normal(size=(B, T + 1, A, 1)).astype(np.float32) * 3.0,
    )
    data["avail_actions"][0, 1, 0, (data["actions"][0, 1, 0, 0] + 1) % args.n_actions] = 0
    term = np.zeros((B, T + 1, A, 1), dtype=np.uint8)
    term[1, T - 2:, 0] = 1
    term[5, 4:, 0] = 1
    data["terminated"] = term
    batch.update(data, bs=slice(None), ts=slice(None))
    learner.insert_episode_batch(batch)
    rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
               data={k: torch.as_tensor(v) for k, v in data.items()},
               actors_before=[small(sd_clone(m)) for m in mac.agents], critics_before=[small(sd_clone(m)) for m in mac.critics])
    before = [sd_clone(m) for m in list(mac.agents) + list(mac.critics)]
    seed = 1618
    torch.manual_seed(seed)
    learner.train(t_env=0)
    torch.manual_seed(seed)
    n = args.batch_size * T
    rec["perms"] = torch.stack([torch.stack([torch.randperm(n) for _ in range(args.ppo_epoch)]) for _ in range(A)])
    rec["actors_after"] = [trained(sd_clone(m), b, ACTOR_TRAINABLE) for m, b in zip(mac.agents, before)]
    rec["critics_after"] = [trained(sd_clone(m), b, CRITIC_TRAINABLE) for m, b in zip(mac.critics, before[A:])]
    rec["stats"] = dict(logger.stats)
    rec["opt_step"] = int(next(iter(learner.actor_optimizers[0].state_dict()["state"].values()))["step"])
    assert rec["opt_step"] == args.ppo_epoch * args.num_mini_batch
    print("learner minibatch", {k.split("_H_")[-1]: round(v, 6) for k, v in logger.stats.items()})
    torch.save(rec, os.path.join(HERE, "learner_minibatch.pt"))


if __name__ == "__main__":
    main()
