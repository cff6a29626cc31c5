"""CPU oracle of the fully-connected behaviour module (iPLAN-FC; reference nova/behavior_FC_policy.py,
nova/behavior_FC_net.py), built from the window, clip and Adam helpers of oracle/iplan_oracle.py.  It specifies the
arithmetic of ``iplan_b200.nova.behavior_FC_policy.Behavior_policy`` (kernels csrc/behavior_fc.cu), runs in the dtype of
its inputs (float64 for the GPU parity tests), and is pinned to recorded calls of the reference by
tests/test_beh_fc_cpu.py (fixtures tests/golden/behavior_learn_fc_{mpe,highway}.pt)."""
import torch

from oracle.iplan_oracle import AdamState, behavior_windows, clip_grads

FC_ENCODER_KEYS = ["linear_1.weight", "linear_1.bias", "linear_2.weight", "linear_2.bias", "out.weight", "out.bias"]
FC_DECODER_KEYS = ["decoder." + k for k in FC_ENCODER_KEYS]


def fc_encoder(p, x):
    """Encoder_3FC.forward (:16-20): x [..., W*o] -> soft-max latent [..., L]."""
    h = torch.tanh(x @ p["linear_1.weight"].t() + p["linear_1.bias"])
    h = torch.tanh(h @ p["linear_2.weight"].t() + p["linear_2.bias"])
    return torch.softmax(h @ p["out.weight"].t() + p["out.bias"], dim=-1)


def fc_decoder(dp, x, latent):
    """LILI_Latent_Decoder.forward (:46-60) + Decoder_3FC.forward (:33-37): [x | latent] -> prediction [..., W*o]."""
    h = torch.cat([x, latent], dim=-1)
    h = torch.tanh(h @ dp["decoder.linear_1.weight"].t() + dp["decoder.linear_1.bias"])
    h = torch.tanh(h @ dp["decoder.linear_2.weight"].t() + dp["decoder.linear_2.bias"])
    return h @ dp["decoder.out.weight"].t() + dp["decoder.out.bias"]


def fc_latent_update(enc_params, history):
    """Behavior_policy.latent_update (:80-106): history [B,A,N,W,o] -> latent [B,A,N,L]; no state, no soft update."""
    hist = torch.as_tensor(history)
    B, A, N, W, o = hist.shape
    return torch.stack([fc_encoder(enc_params[a], hist[:, a].reshape(B, N, W * o)) for a in range(A)], dim=1)


def behavior_learn_fc_agent(enc_p, dec_p, history, mask, args, opt=None):
    """One agent-net's share of ``learn`` (:168-230).  history [B,T,N,o] (the batch without its last step), mask [B,T]
    (``terminated`` of the agent).  For j = 0 .. T-2-W: the decoder reads the window ending at j with latent_{j-1}
    (latent_{-1} = 0), then latent_j = encoder(window ending at j); the target is the window ending at j + 1 (NOT the
    second output of behavior_windows, which is the W rows after j).  The reference builds a next-window mask from
    ``mask`` but its loop writes the current-window mask twice (:135-140), so the next-window mask it multiplies by stays
    all ones; ``mask`` is accepted and has no effect, as there.  loss = mean_j sum |next - pred| / (B N W o + 1e-10) o N.
    Encoder and decoder gradients clipped separately, then one Adam step over both.  Updates the dicts in place;
    returns (stats, AdamState)."""
    B, T, N, o = history.shape
    W, L = args.max_history_len, args.latent_dim
    n_pos = T - 1 - W
    if n_pos < 1:
        raise RuntimeError(f"episode of {T} steps has no position to train with windows of {W} (T - 1 - W < 1)")
    e_tr = [enc_p[k].requires_grad_(True) for k in FC_ENCODER_KEYS]
    d_tr = [dec_p[k].requires_grad_(True) for k in FC_DECODER_KEYS]
    latent = torch.zeros(B, N, L, dtype=history.dtype)
    m_next = torch.ones(B, N, W, o, dtype=history.dtype)          # the reference's mask_over_next_traj: never written
    loss = 0.0
    for j in range(n_pos):
        curr = behavior_windows(history, j, W)[0].reshape(B, N, W * o)
        nxt = behavior_windows(history, j + 1, W)[0].reshape(B, N, W * o)
        pred = fc_decoder(dec_p, curr, latent)
        latent = fc_encoder(enc_p, curr)
        err = (nxt - pred).abs() * m_next.reshape(B, N, W * o)
        loss = loss + err.sum() / (m_next.sum() + 1e-10) * o * N
    loss = loss / n_pos
    grads = torch.autograd.grad(loss, e_tr + d_tr)
    g_e, n_e = clip_grads(list(grads[:len(e_tr)]), args.max_grad_norm)
    g_d, n_d = clip_grads(list(grads[len(e_tr):]), args.max_grad_norm)
    opt = opt or AdamState(e_tr + d_tr, args.lr_behavior, args.optim_eps)
    with torch.no_grad():
        opt.step(g_e + g_d)
    for t in e_tr + d_tr:
        t.requires_grad_(False)
    keys = ["enc:" + k for k in FC_ENCODER_KEYS] + ["dec:" + k for k in FC_DECODER_KEYS]
    return dict(behavior_loss=float(loss.detach()), enc_grad_norm=float(n_e), dec_grad_norm=float(n_d),
                grads=dict(zip(keys, [g.detach() for g in grads])),
                clipped=dict(zip(keys, [g.detach() for g in g_e + g_d]))), opt
