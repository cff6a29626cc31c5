"""CPU oracle of the hard-update behaviour learner (iPLAN-Hard; reference nova/behavior_policy.py:119-215), built from
the encoder / decoder / clip / Adam helpers of oracle/iplan_oracle.py.  It specifies the arithmetic of
``iplan_b200.nova.behavior_policy.Behavior_policy.learn`` and is pinned to a recorded call of the reference by
tests/test_beh_hard_oracle.py (fixture tests/golden/behavior_learn_hard.pt)."""
import torch

from oracle.iplan_oracle import (BEH_ENCODER_KEYS, DECODER_KEYS, AdamState, behavior_decoder, behavior_encoder,
                                 clip_grads)


def behavior_learn_hard_agent(enc_p, dec_p, history, mask, keep, args, opt=None):
    """One agent-net's share of the hard-update ``learn``.  history [B,T,N,o] (the batch without its last step),
    mask [B,T] (``terminated`` on Highway, ``1 - terminated`` on MPE, :146-149), keep [T/W-1, B*N, W, Hd].
    The episode is T/W windows of W steps (T % W != 0 raises, as the reference's reshape does, :142).  For
    j = 0 .. T/W-2 the decoder reads window j with latent_j (latent_0 = 0) and the carried decoder hidden, then the encoder
    reads window j from the carried encoder hidden and its soft-max output is latent_{j+1} (no soft update).  Targets are
    windows 1 .. T/W-1, weighted by the mask's first (T/W-1) W rows (:144-152), i.e. target row t by mask[t - W].
    loss = sum |next - pred| m / (N o sum m + 1e-10) o N (:184-186).  Encoder and decoder gradients are clipped
    separately, then one Adam step over both.  Updates the dicts in place; returns (stats, AdamState)."""
    B, T, N, o = history.shape
    W, L = args.max_history_len, args.latent_dim
    if T % W != 0:
        raise RuntimeError(f"episode of {T} steps is not a whole number of windows of {W}")
    n_win = T // W
    if n_win < 2:
        raise RuntimeError(f"episode of {T} steps has fewer than two windows of {W}")
    cut = (n_win - 1) * W
    e_tr = [enc_p[k].requires_grad_(True) for k in BEH_ENCODER_KEYS]
    d_tr = [dec_p[k].requires_grad_(True) for k in DECODER_KEYS]
    wins = history.reshape(B, n_win, W, N, o)
    latent = torch.zeros(B, N, L, dtype=history.dtype)
    eh = torch.zeros(B * N, args.encoder_rnn_dim, dtype=history.dtype)
    dh = torch.zeros(B * N, args.decoder_rnn_dim, dtype=history.dtype)
    preds = []
    for j in range(n_win - 1):
        curr = wins[:, j].permute(0, 2, 1, 3)                                         # [B, N, W, o]
        pred, dh = behavior_decoder(dec_p, curr, latent, dh, keep[j], args.decoder_dropout)
        preds.append(pred.permute(0, 2, 1, 3))                                        # [B, W, N, o]
        eh, latent = behavior_encoder(enc_p, curr.reshape(B * N, W, o), eh)
        latent = latent.view(B, N, L)
    nxt = wins[:, 1:].reshape(B, cut, N, o)
    pred = torch.cat(preds, dim=1)
    m = mask[:, :cut].to(history.dtype).view(B, cut, 1, 1).expand(B, cut, N, o)
    loss = ((nxt - pred).abs() * m).sum() / (m.sum() + 1e-10) * o * N
    grads = torch.autograd.grad(loss, e_tr + d_tr)
    g_e, n_e = clip_grads(list(grads[:len(e_tr)]), args.max_grad_norm)
    g_d, n_d = clip_grads(list(grads[len(e_tr):]), args.max_grad_norm)
    opt = opt or AdamState(e_tr + d_tr, args.lr_behavior, args.optim_eps)
    with torch.no_grad():
        opt.step(g_e + g_d)
    for t in e_tr + d_tr:
        t.requires_grad_(False)
    keys = ["enc:" + k for k in BEH_ENCODER_KEYS] + ["dec:" + k for k in DECODER_KEYS]
    return dict(behavior_loss=float(loss.detach()), enc_grad_norm=float(n_e), dec_grad_norm=float(n_d),
                grads=dict(zip(keys, [g.detach() for g in grads])),
                clipped=dict(zip(keys, [g.detach() for g in g_e + g_d]))), opt
