#!/usr/bin/env python
"""Generate tests/golden/behavior_learn_fc_{mpe,highway}.pt by RUNNING THE REFERENCE'S fully-connected behaviour module
(nova/behavior_FC_policy.Behavior_policy, selected by ``behavior_fully_connected: True``, reference run_ippo.py:200-203)
on the CPU.  Needs the reference checkout; writes only those two files, so the other fixtures stay as they are.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_fc.py

Per case: one ``learn`` call, a save_models into a temporary directory (key names and shapes of the three files are
recorded), then three ``latent_update`` calls with the trained encoder.  The inputs come from beh_fc_inputs.fc_inputs
(seeded), which also documents what is stored.
  mpe:     A=3, N=6,  B=3, T=40 (29 positions, 522 rows per agent-net)
  highway: A=2, N=55, B=2, T=30 (19 positions, 2090 rows per agent-net: a ragged last tile of 42 rows)"""
import os
import tempfile

import numpy as np
import torch

from beh_fc_inputs import CASES, fc_inputs, fixture_path
from make_golden import HERE, NullLogger, make_scheme, ref_args, sd_clone


def golden_behavior_learn_fc():
    from nova.behavior_FC_policy import Behavior_policy
    from components.episode_buffer import EpisodeBatch

    for name, (env, over, _) in CASES.items():
        args = ref_args(env, **over)
        A, B, T = args.n_agents, args.batch_size_run, args.episode_limit
        x = fc_inputs(name, args)
        logger = NullLogger()
        pol = Behavior_policy(args, logger)
        for a in range(A):
            pol.behavior_encoder[a].load_state_dict(x["enc"][a])
            pol.behavior_decoder[a].load_state_dict(x["dec"][a])
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        batch.update({"history": x["history"].numpy(), "terminated": x["terminated"].numpy()}, bs=slice(None), ts=slice(None))
        b_loss, s_loss, t_loss = pol.learn(batch, t_env=0)
        after = [{**{"enc:" + k: v for k, v in sd_clone(pol.behavior_encoder[a]).items()},
                  **{"dec:" + k: v for k, v in sd_clone(pol.behavior_decoder[a]).items()}} for a in range(A)]
        before = [{**{"enc:" + k: v for k, v in x["enc"][a].items()}, **{"dec:" + k: v for k, v in x["dec"][a].items()}} for a in range(A)]
        with tempfile.TemporaryDirectory() as d:
            pol.save_models(d)
            enc_sd = torch.load(os.path.join(d, "behavior_encoder_0.th"), weights_only=False)
            dec_sd = torch.load(os.path.join(d, "behavior_decoder_0.th"), weights_only=False)
            opt_sd = torch.load(os.path.join(d, "behavior_optimizer_0_opt.th"), weights_only=False)
        files = dict(encoder=[(k, tuple(v.shape)) for k, v in enc_sd.items()], decoder=[(k, tuple(v.shape)) for k, v in dec_sd.items()],
                     optimizer={pid: tuple(s["exp_avg"].shape) for pid, s in opt_sd["state"].items()},
                     optimizer_params=list(opt_sd["param_groups"][0]["params"]))
        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   behavior_loss=[float(v) for v in b_loss], total_loss=[float(v) for v in t_loss],
                   stability_loss=list(s_loss), stats=dict(logger.stats), files=files,
                   delta_after=[{k: (after[a][k] - before[a][k]).half() for k in before[a]} for a in range(A)],
                   grads0={**{"enc:" + k: v.grad.detach().clone() for k, v in pol.behavior_encoder[0].named_parameters()},
                           **{"dec:" + k: v.grad.detach().clone() for k, v in pol.behavior_decoder[0].named_parameters()}})
        rec["latent_out"] = []
        for t in range(3):
            new, hid = pol.latent_update(x["windows"][t].numpy(), None, None)
            assert hid is None
            rec["latent_out"].append(torch.as_tensor(np.asarray(new, dtype=np.float32)))
        path = fixture_path(HERE, name)
        torch.save(rec, path)
        print("behavior.learn (fc)", name, [round(float(v), 6) for v in b_loss], os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_behavior_learn_fc()
