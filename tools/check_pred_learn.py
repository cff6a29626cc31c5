"""Prediction_policy.learn on the GPU (kernel csrc/pred_learn.cu) against the reference's recorded ``learn`` call
(tests/golden/prediction_learn.pt: sampled indices, Gumbel noise and dropout masks replayed):

    timeout 120 python tools/check_pred_learn.py

Prints, per case and tensor, the relative difference of the raw gradients to the oracle's (autograd) and of the
post-step weights to the reference's, so that a partial failure localises the faulty phase of the kernel."""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iplan_b200.components.episode_buffer import EpisodeBatch            # noqa: E402
from iplan_b200.components.transforms import OneHot                      # noqa: E402
from iplan_b200.config import make_args                                  # noqa: E402
from iplan_b200.nova.prediction_policy import Prediction_policy          # noqa: E402
from oracle import iplan_oracle as O                                     # noqa: E402

# every raw gradient tensor against the oracle, relative to the tensor's largest entry: both recorded cases stay
# below 1e-5 (worst 9.4e-6, on an NVIDIA H100 80GB HBM3); the kernel's float atomics vary the last bits run to run
GRAD_REL = 2e-5


def scheme_for(args):
    scheme = {
        "state": {"vshape": args.state_shape}, "obs": {"vshape": args.obs_shape, "group": "agents"},
        "actions": {"vshape": (1,), "group": "agents", "dtype": torch.long},
        "rnn_states_actors": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "rnn_states_critics": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "history": {"vshape": (args.max_vehicle_num, args.obs_shape_single,), "group": "agents"},
        "behavior_latent": {"vshape": (args.max_vehicle_num, args.latent_dim,), "group": "agents"},
        "attention_latent": {"vshape": (args.max_vehicle_num, args.attention_dim,), "group": "agents"},
        "avail_actions": {"vshape": (args.n_actions,), "group": "agents", "dtype": torch.int},
        "reward": {"vshape": (1,), "group": "agents"}, "speed": {"vshape": (1,), "group": "agents"},
        "terminated": {"vshape": (1,), "group": "agents", "dtype": torch.uint8},
    }
    return scheme, {"agents": args.n_agents}, {"actions": ("actions_onehot", [OneHot(out_dim=args.n_actions)])}


def run(case):
    g = torch.load(os.path.join(ROOT, "tests", "golden", "prediction_learn.pt"), weights_only=False)[case]
    args = make_args(g["args"].get("env", "highway"))
    for k, v in g["args"].items():
        setattr(args, k, v)
    args.use_cuda, args.device = True, "cuda"
    A, N = args.n_agents, args.max_vehicle_num
    d = g["data"]
    B, T1 = d["history"].shape[:2]
    scheme, groups, pre = scheme_for(args)
    batch = EpisodeBatch(scheme, groups, B, T1, preprocess=pre, device="cuda")
    batch.update({k: v.numpy() for k, v in d.items()}, bs=slice(None), ts=slice(None))
    pol = Prediction_policy(args, None)
    for a in range(A):
        pol.pred_GAT[a].load_state_dict(g["gat_before"][a])
        pol.pred_decoder[a].load_state_dict(g["dec_before"][a])
    P, pl = args.pred_batch_size, args.pred_length
    keep = torch.stack([k.view(pl, P, N, -1).permute(1, 0, 2, 3) for k in g["dropout_keep"]]).to(torch.uint8)   # [A,P,pl,N,32]
    pol.debug_learn = dict(select_idx=g["select_idx"], gumbel=torch.stack(g["gumbel"]), keep=keep)
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    ok = True
    hist, att, beh = d["history"][:, :-1], d["attention_latent"][:, :-1], d["behavior_latent"][:, :-1]
    flag = d["terminated"][:, :-1, :, 0]
    oargs = SimpleNamespace(**g["args"])
    for a in range(A):
        gp = {k: v.clone() for k, v in g["gat_before"][a].items()}
        dp = {k: v.clone() for k, v in g["dec_before"][a].items()}
        ref, _ = O.prediction_learn_agent(gp, dp, hist[:, :, a], att[:, :, a], beh[:, :, a], flag[:, :, a],
                                          g["select_idx"][a], g["gumbel"][a], g["dropout_keep"][a], oargs)
        dl = abs(float(losses[a]) - g["losses"][a]) / abs(g["losses"][a])
        print(f"[{case} a={a}] loss cuda {float(losses[a]):.6f} reference {g['losses'][a]:.6f} (rel {dl:.2e})")
        ok &= dl < 1e-4
        for kind, stack, flat in (("gat", pol.stack, pol.last_grads["gat"]), ("dec", pol.dec_stack, pol.last_grads["dec"])):
            for name, (off, shape) in stack.named_offsets().items():
                n = 1
                for s_ in shape:
                    n *= s_
                mine = flat[a, off:off + n].view(shape).cpu()
                want = ref["grads"][name]
                rel = float((mine - want).abs().max() / (want.abs().max() + 1e-12))
                flagged = "" if rel < GRAD_REL else "   <-- MISMATCH"
                print(f"    grad {kind}:{name:34s} rel {rel:.2e}{flagged}")
                ok &= rel < GRAD_REL
        after = {**{"gat:" + k: v for k, v in pol.pred_GAT[a].state_dict().items()}, **{"dec:" + k: v for k, v in pol.pred_decoder[a].state_dict().items()}}
        want = {**{"gat:" + k: v for k, v in g["gat_after"][a].items()}, **{"dec:" + k: v for k, v in g["dec_after"][a].items()}}
        worst = max(float((after[k].cpu() - want[k]).abs().max()) for k in want)
        print(f"    max |weight - reference| after the step: {worst:.2e}")
        ok &= worst < 1e-6
    return ok


if __name__ == "__main__":
    res = [run(c) for c in ("mpe", "highway")]
    print("OK" if all(res) else "MISMATCH")
