"""Inputs and loader of the hard-update behaviour fixtures (behavior_learn_hard_{mpe,highway}.pt).

The inputs of the recorded reference calls (initial weights, episodes, terminations, rollout windows) are drawn here from
fixed seeds with torch's CPU generator, so that only the reference's outputs are stored: the dropout masks as packed bits,
the losses, agent-net 0's clipped gradients, every agent-net's post-step weight change (float16: a first Adam step moves a
weight by at most lr = 1e-4, so this is exact to ~5e-8) and the rollout outputs.  ``load_hard_case`` reassembles
everything into one dict."""
import os

import numpy as np
import torch

CASES = {   # name: (env, reference config overrides, seed)
    "mpe": ("MPE", dict(episode_length=40, batch_size_run=3, soft_update_enable=False), 61),
    "highway": ("highway", dict(n_agents=2, n_other_vehicles=53, episode_limit=30, batch_size_run=2, soft_update_enable=False), 62),
}
ENC_SHAPES = lambda o, L, E: {"linear.weight": (E, o), "linear.bias": (E,), "rnn.weight_ih_l0": (3 * E, E),
                              "rnn.weight_hh_l0": (3 * E, E), "rnn.bias_ih_l0": (3 * E,), "rnn.bias_hh_l0": (3 * E,),
                              "out.weight": (L, E), "out.bias": (L,)}
DEC_SHAPES = lambda o, L, H: {"decoder.linear.weight": (H, o + L), "decoder.linear.bias": (H,),
                              "decoder.rnn.weight_ih_l0": (3 * H, H), "decoder.rnn.weight_hh_l0": (3 * H, H),
                              "decoder.rnn.bias_ih_l0": (3 * H,), "decoder.rnn.bias_hh_l0": (3 * H,),
                              "decoder.out.weight": (o, H), "decoder.out.bias": (o,)}


def _uniform(g, shape, bound):
    return (torch.rand(shape, generator=g) * 2 - 1) * bound


def hard_inputs(name, args):
    """Initial weights (U(-1/sqrt(k), 1/sqrt(k)), k = last dimension), episodes [B,T+1,A,N,o] (column 0 = 1, slots
    >= 3 + 2t empty at step t), terminations [B,T+1,A,1] placed where the one-window mask lag changes the loss, and three
    rollout windows [B,A,N,W,o] with random previous latents [B,A,N,L]."""
    env, _, seed = CASES[name]
    A, N, o, L, W, B = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.max_history_len, args.batch_size_run
    T = args.episode_limit
    g = torch.Generator().manual_seed(seed)
    enc = [{k: _uniform(g, s, s[-1] ** -0.5) for k, s in ENC_SHAPES(o, L, args.encoder_rnn_dim).items()} for _ in range(A)]
    dec = [{k: _uniform(g, s, s[-1] ** -0.5) for k, s in DEC_SHAPES(o, L, args.decoder_rnn_dim).items()} for _ in range(A)]
    hist = _uniform(g, (B, T + 1, A, N, o), 1.0)
    hist[..., 0] = 1.0
    for t in range(T + 1):
        hist[:, t, :, min(N, 3 + 2 * t):] = 0.0
    term = torch.zeros(B, T + 1, A, 1, dtype=torch.uint8)
    term[0, 17:, 0] = 1
    term[B - 1, 24:, A - 1] = 1
    if env != "MPE":
        term = 1 - term            # highway: the flag is the mask itself (reference nova/behavior_policy.py:146-149)
    windows, prevs = [], []
    for t in range(3):
        w = _uniform(g, (B, A, N, W, o), 1.0)
        w[..., 0] = 1.0
        w[:, :, min(N, 6 + 4 * t):] = 0.0
        windows.append(w)
        prevs.append(torch.softmax(torch.randn(B, A, N, L, generator=g), dim=-1))
    return dict(enc=enc, dec=dec, history=hist, terminated=term, windows=windows, prevs=prevs)


def fixture_path(golden_dir, name):
    return os.path.join(golden_dir, f"behavior_learn_hard_{name}.pt")


def load_hard_case(golden_dir, name):
    """The recorded case with its inputs: args, data {history, terminated}, enc_before / dec_before / enc_after /
    dec_after [A] state dicts, dropout_keep [A] bool [n_pos, B*N, W, 64], behavior_loss [A], stats, grads0 (agent-net
    0's clipped gradients, keys "enc:" / "dec:" + name), latent_steps [3] {window, hid_in, prev, latent, hid_out}."""
    from types import SimpleNamespace
    r = torch.load(fixture_path(golden_dir, name), weights_only=False)
    args = SimpleNamespace(**r["args"])
    x = hard_inputs(name, args)
    keep = [torch.from_numpy(np.unpackbits(p.numpy(), count=int(np.prod(r["keep_shape"])))).view(*r["keep_shape"]).bool()
            for p in r["keep_bits"]]
    enc_after = [{k: v + r["delta_after"][a]["enc:" + k].float() for k, v in x["enc"][a].items()} for a in range(args.n_agents)]
    dec_after = [{k: v + r["delta_after"][a]["dec:" + k].float() for k, v in x["dec"][a].items()} for a in range(args.n_agents)]
    steps, hid = [], torch.zeros(r["latent_out"][0]["hid_out"].shape)
    for t, out in enumerate(r["latent_out"]):
        steps.append(dict(window=x["windows"][t], hid_in=hid, prev=x["prevs"][t], latent=out["latent"], hid_out=out["hid_out"]))
        hid = out["hid_out"]
    return dict(args=r["args"], data=dict(history=x["history"], terminated=x["terminated"]), enc_before=x["enc"],
                dec_before=x["dec"], enc_after=enc_after, dec_after=dec_after, dropout_keep=keep,
                behavior_loss=r["behavior_loss"], stats=r["stats"], grads0=r["grads0"], latent_steps=steps)
