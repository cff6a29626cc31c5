"""BASELINE.json configs[4] — GAT_Net.forward at hidden width 128, 16 slots (the synthetic GAT + GRU microbench):
the CUDA path (iplan_b200/nova/gat128.py: library GEMMs + the wgmma recurrence with W_hh in shared memory + the
attention / gate kernels) against the CPU oracle's ``gat_forward`` (oracle/iplan_oracle.py, generic in the widths, pinned
to the reference's GAT_Net by tests/test_oracle_golden.py) with explicit Gumbel noise.  Tolerance 1e-4 (north_star)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


@pytest.mark.parametrize("A,items", [(2, 5), (3, 64)])
def test_gat128_vs_oracle(A, items):
    """Odd / even item counts, several agent-nets; dl, hard gates and the output."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from iplan_b200.nova.gat128 import GAT128, H, N
    from oracle import iplan_oracle as O
    torch.manual_seed(7 + items)
    net = GAT128(A, seed=3)
    with torch.no_grad():                       # larger recurrent weights: make the gates and the hard attention non-trivial
        for k in ("hard_bi_GRU.weight_hh_l0", "hard_bi_GRU.weight_hh_l0_reverse", "hard_encoding.weight"):
            net.p[k].mul_(2.0)
    x = (torch.rand(A, items, N, H, device="cuda") * 2 - 1).contiguous()
    hp = torch.tanh(torch.randn(A, items, N, H, device="cuda")).contiguous()
    gum = -torch.log(torch.empty(A, items, N, N - 1, 2, device="cuda").exponential_())
    out = net.forward(x, hp, gumbel=gum)
    torch.cuda.synchronize()
    worst = 0.0
    for a in range(A):
        sd = net.state_dict(a)
        ref, parts = O.gat_forward(sd, x[a].cpu(), hp[a].cpu().reshape(items * N, H), gum[a].cpu(), return_parts=True)
        d = float((out[a].cpu().reshape(items * N, H) - ref).abs().max())
        # the per-edge logit differences the recurrence kernel produced: dl[item][dir][s][i] summed over directions + bias
        dl = net._buf["dl"][a].cpu()                                     # [items, 2, 15, 16]
        mine = (dl[:, 0] + dl[:, 1]).permute(0, 2, 1) + float(sd["hard_encoding.bias"][1] - sd["hard_encoding.bias"][0])
        theirs = parts["logits"][..., 1] - parts["logits"][..., 0]       # [items, 16, 15]
        dlg = float((mine - theirs).abs().max())
        print(f"[gat128 A={A} items={items} a={a}] max|out - oracle| = {d:.3e}   max|logit diff - oracle| = {dlg:.3e} "
              f"(|logit diff| max {float(theirs.abs().max()):.2f})")
        worst = max(worst, d)
        assert dlg < 1e-4
    assert worst < 1e-4
