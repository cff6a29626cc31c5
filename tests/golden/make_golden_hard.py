#!/usr/bin/env python
"""Generate tests/golden/behavior_learn_hard_{mpe,highway}.pt by RUNNING THE REFERENCE'S hard-update behaviour module
(nova/behavior_policy.Behavior_policy, selected by ``soft_update_enable: False``, reference run_ippo.py:200-209) on the
CPU.  Needs the reference checkout; writes only those two files, so the other fixtures stay as they are.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_hard.py

Per case: one ``learn`` call with the decoder's dropout read off a forward hook (as make_golden.golden_behavior_learn
does for the soft update), then three consecutive ``latent_update`` calls with the encoder hidden state carried.  The
inputs come from beh_hard_inputs.hard_inputs (seeded), which also documents what is stored.
  mpe:     A=3, N=6,  B=3, T=40 (4 windows of 10, 3 trained)
  highway: A=2, N=55, B=2, T=30 (3 windows, 2 trained; 110 chains per agent-net)"""
import os

import numpy as np
import torch

from beh_hard_inputs import CASES, fixture_path, hard_inputs
from make_golden import HERE, NullLogger, make_scheme, ref_args, sd_clone


def golden_behavior_learn_hard():
    from nova.behavior_policy import Behavior_policy
    from components.episode_buffer import EpisodeBatch

    for name, (env, over, _) in CASES.items():
        args = ref_args(env, **over)
        A, B, T = args.n_agents, args.batch_size_run, args.episode_limit
        x = hard_inputs(name, args)
        logger = NullLogger()
        pol = Behavior_policy(args, logger)
        for a in range(A):
            pol.behavior_encoder[a].load_state_dict(x["enc"][a])
            pol.behavior_decoder[a].load_state_dict(x["dec"][a])
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        batch.update({"history": x["history"].numpy(), "terminated": x["terminated"].numpy()}, bs=slice(None), ts=slice(None))
        drop = [[] for _ in range(A)]
        hooks = []
        for i in range(A):
            def hook(mod, inp, out, i=i):
                assert bool((inp[0].detach() != 0).all())
                drop[i].append((out.detach() != 0).clone())
            hooks.append(pol.behavior_decoder[i].decoder.dropout.register_forward_hook(hook))
        torch.manual_seed(9091)
        try:
            b_loss = pol.learn(batch, t_env=0)
        finally:
            for h in hooks:
                h.remove()
        keep = [torch.stack(m) for m in drop]
        after = [{**{"enc:" + k: v for k, v in sd_clone(pol.behavior_encoder[a]).items()},
                  **{"dec:" + k: v for k, v in sd_clone(pol.behavior_decoder[a]).items()}} for a in range(A)]
        before = [{**{"enc:" + k: v for k, v in x["enc"][a].items()}, **{"dec:" + k: v for k, v in x["dec"][a].items()}} for a in range(A)]
        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   keep_shape=tuple(keep[0].shape),
                   keep_bits=[torch.from_numpy(np.packbits(k.numpy().reshape(-1))) for k in keep],
                   behavior_loss=[float(v) for v in b_loss], stats=dict(logger.stats),
                   delta_after=[{k: (after[a][k] - before[a][k]).half() for k in before[a]} for a in range(A)],
                   grads0={**{"enc:" + k: v.grad.detach().clone() for k, v in pol.behavior_encoder[0].named_parameters()},
                           **{"dec:" + k: v.grad.detach().clone() for k, v in pol.behavior_decoder[0].named_parameters()}})
        # three rollout steps with the trained encoder; prev_latent is random (the hard update ignores it)
        hid = np.zeros((B, 1, A, args.max_vehicle_num, args.encoder_rnn_dim), dtype=np.float32)
        rec["latent_out"] = []
        for t in range(3):
            new, hid_t = pol.latent_update(x["windows"][t].numpy(), hid, x["prevs"][t].numpy())
            rec["latent_out"].append(dict(latent=torch.as_tensor(np.asarray(new, dtype=np.float32)), hid_out=hid_t.detach().clone()))
            hid = hid_t.detach().numpy().copy()
        path = fixture_path(HERE, name)
        torch.save(rec, path)
        print("behavior.learn (hard)", name, [round(float(v), 6) for v in b_loss], "windows trained:", len(drop[0]),
              os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_behavior_learn_hard()
