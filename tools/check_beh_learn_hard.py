"""Behavior_policy.learn of the hard-update variant (iPLAN-Hard; iplan_b200/nova/behavior_policy.py, kernels
csrc/beh_learn_tile.cu with the window geometry (W, 0)) against the reference's recorded ``learn`` call
(tests/golden/behavior_learn_hard_{mpe,highway}.pt, dropout masks replayed):

    timeout 200 python tools/check_beh_learn_hard.py

Prints, per case and tensor, the relative difference of the clipped gradients to the oracle's (autograd,
tools/beh_hard_oracle.py) and of the post-step weights to the reference's, so that a partial failure localises the faulty
phase of the kernels."""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iplan_b200.components.episode_buffer import EpisodeBatch            # noqa: E402
from iplan_b200.config import make_args                                  # noqa: E402
from iplan_b200.nova.behavior_policy import Behavior_policy              # noqa: E402
from tools.beh_hard_oracle import behavior_learn_hard_agent              # noqa: E402
from tools.check_pred_learn import scheme_for                            # noqa: E402


def load_case(case):
    golden = os.path.join(ROOT, "tests", "golden")
    if golden not in sys.path:
        sys.path.insert(0, golden)
    from beh_hard_inputs import load_hard_case
    return load_hard_case(golden, case)


def gpu_args(g):
    args = make_args(g["args"].get("env", "highway"))
    for k, v in g["args"].items():
        setattr(args, k, v)
    args.use_cuda, args.device = True, "cuda"
    return args


def keep_for_gpu(keeps, B, N, W):
    """Per-agent [n_pos, B*N, W, 64] dropout masks (the oracle's layout) -> uint8 [A, B, n_pos, N, W, 64]."""
    return torch.stack([k.reshape(k.shape[0], B, N, W, -1).permute(1, 0, 2, 3, 4) for k in keeps]).to(torch.uint8)


def compare(pol, data, keeps, oargs, enc_before, dec_before, losses, want_after=None, tag=""):
    """Gradients and losses of the last ``pol.learn`` against the oracle run from the same weights; post-step weights
    against ``want_after`` (per agent: {"enc:"/"dec:" + name: tensor}) or, when None, against the oracle's."""
    hist = data["history"][:, :-1]
    term = data["terminated"][:, :-1, :, 0].float()
    ok = True
    for a in range(oargs.n_agents):
        mask = 1 - term[:, :, a] if oargs.env == "MPE" else term[:, :, a]
        ep = {k: v.clone() for k, v in enc_before[a].items()}
        dp = {k: v.clone() for k, v in dec_before[a].items()}
        ref, _ = behavior_learn_hard_agent(ep, dp, hist[:, :, a], mask, keeps[a], oargs)
        db = abs(float(losses[a]) - ref["behavior_loss"]) / abs(ref["behavior_loss"])
        print(f"[{tag} a={a}] behavior loss cuda {float(losses[a]):.6f} oracle {ref['behavior_loss']:.6f} (rel {db:.2e})")
        ok &= db < 1e-4
        # the oracle returns the gradients as clipped by the reference; clip ours the same way per group
        for kind, stack, flat in (("enc", pol.stack, pol.last_grads["enc"]), ("dec", pol.dec_stack, pol.last_grads["dec"])):
            mine_all = {name: flat[a, off:off + max(1, int(torch.tensor(shape).prod()))].view(shape).cpu()
                        for name, (off, shape) in stack.named_offsets().items()}
            total = torch.sqrt(sum((v ** 2).sum() for v in mine_all.values()))
            coef = min(1.0, float(oargs.max_grad_norm) / (float(total) + 1e-6))
            for name, mine in mine_all.items():
                want = ref["clipped"][kind + ":" + name]
                rel = float((mine * coef - want).abs().max() / (want.abs().max() + 1e-12))
                flagged = "" if rel < 1e-3 else "   <-- MISMATCH"
                if a == 0 or flagged:
                    print(f"    grad {kind}:{name:28s} rel {rel:.2e}{flagged}")
                ok &= rel < 1e-3
        after = {**{"enc:" + k: v for k, v in pol.behavior_encoder[a].state_dict().items()},
                 **{"dec:" + k: v for k, v in pol.behavior_decoder[a].state_dict().items()}}
        want = want_after[a] if want_after is not None else {**{"enc:" + k: v for k, v in ep.items()}, **{"dec:" + k: v for k, v in dp.items()}}
        worst = max(float((after[k].cpu() - want[k]).abs().max()) for k in want)
        print(f"    max |weight - {'reference' if want_after is not None else 'oracle'}| after the step: {worst:.2e}")
        ok &= worst < 1e-6
    return ok


def run(case):
    g = load_case(case)
    args = gpu_args(g)
    A, N, W = args.n_agents, args.max_vehicle_num, args.max_history_len
    d = g["data"]
    B, T1 = d["history"].shape[:2]
    scheme, groups, pre = scheme_for(args)
    batch = EpisodeBatch(scheme, groups, B, T1, preprocess=pre, device="cuda")
    batch.update({k: v.numpy() for k, v in d.items()}, bs=slice(None), ts=slice(None))
    pol = Behavior_policy(args, None)
    for a in range(A):
        pol.behavior_encoder[a].load_state_dict(g["enc_before"][a])
        pol.behavior_decoder[a].load_state_dict(g["dec_before"][a])
    pol.debug_keep = keep_for_gpu(g["dropout_keep"], B, N, W)
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    ok = len(losses) == A
    for a in range(A):
        db = abs(float(losses[a]) - g["behavior_loss"][a]) / abs(g["behavior_loss"][a])
        print(f"[{case} a={a}] behavior loss cuda {float(losses[a]):.6f} reference {g['behavior_loss'][a]:.6f} (rel {db:.2e})")
        ok &= db < 1e-4
    want_after = [{**{"enc:" + k: v for k, v in g["enc_after"][a].items()}, **{"dec:" + k: v for k, v in g["dec_after"][a].items()}}
                  for a in range(A)]
    ok &= compare(pol, d, g["dropout_keep"], SimpleNamespace(**g["args"]), g["enc_before"], g["dec_before"], losses,
                  want_after, tag=case)
    return ok


if __name__ == "__main__":
    res = [run(c) for c in ("mpe", "highway")]
    print("OK" if all(res) else "MISMATCH")
