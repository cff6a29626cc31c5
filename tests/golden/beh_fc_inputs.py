"""Inputs and loader of the iPLAN-FC behaviour fixtures (behavior_learn_fc_{mpe,highway}.pt).

The inputs of the recorded reference calls (initial weights, episodes, terminations, rollout windows) are drawn here from
fixed seeds with torch's CPU generator, so that only the reference's outputs are stored: the losses, agent-net 0's
clipped gradients, every agent-net's post-step weight change (float16: a first Adam step moves a weight by at most
lr = 1e-4, so this is exact to ~5e-8), three ``latent_update`` outputs, and the key names and shapes of the saved
encoder, decoder and optimiser files.  ``load_fc_case`` reassembles everything into one dict."""
import os

import torch

CASES = {   # name: (env, reference config overrides, seed)
    "mpe": ("MPE", dict(episode_length=40, batch_size_run=3, behavior_fully_connected=True), 71),
    "highway": ("highway", dict(n_agents=2, n_other_vehicles=53, episode_limit=30, batch_size_run=2,
                                behavior_fully_connected=True), 72),
}
ENC_SHAPES = lambda K0, L, E: {"linear_1.weight": (E, K0), "linear_1.bias": (E,), "linear_2.weight": (E, E),
                               "linear_2.bias": (E,), "out.weight": (L, E), "out.bias": (L,)}
DEC_SHAPES = lambda K0, L, H: {"decoder.linear_1.weight": (H, K0 + L), "decoder.linear_1.bias": (H,),
                               "decoder.linear_2.weight": (H, H), "decoder.linear_2.bias": (H,),
                               "decoder.out.weight": (K0, H), "decoder.out.bias": (K0,)}


def _uniform(g, shape, bound):
    return (torch.rand(shape, generator=g) * 2 - 1) * bound


def fc_inputs(name, args):
    """Initial weights (U(-1/sqrt(k), 1/sqrt(k)), k = last dimension), episodes [B,T+1,A,N,o] (column 0 = 1, slots
    >= 3 + 2t empty at step t), terminations [B,T+1,A,1] (they have no effect on the reference's loss) and three rollout
    windows [B,A,N,W,o]."""
    _, _, seed = CASES[name]
    A, N, o, L, W, B = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.max_history_len, args.batch_size_run
    T, K0 = args.episode_limit, o * W
    g = torch.Generator().manual_seed(seed)
    enc = [{k: _uniform(g, s, s[-1] ** -0.5) for k, s in ENC_SHAPES(K0, L, args.encoder_rnn_dim).items()} for _ in range(A)]
    dec = [{k: _uniform(g, s, s[-1] ** -0.5) for k, s in DEC_SHAPES(K0, L, args.decoder_rnn_dim).items()} for _ in range(A)]
    hist = _uniform(g, (B, T + 1, A, N, o), 1.0)
    hist[..., 0] = 1.0
    for t in range(T + 1):
        hist[:, t, :, min(N, 3 + 2 * t):] = 0.0
    term = torch.zeros(B, T + 1, A, 1, dtype=torch.uint8)
    term[0, 17:, 0] = 1
    term[B - 1, 24:, A - 1] = 1
    windows = []
    for t in range(3):
        w = _uniform(g, (B, A, N, W, o), 1.0)
        w[..., 0] = 1.0
        w[:, :, min(N, 6 + 4 * t):] = 0.0
        windows.append(w)
    return dict(enc=enc, dec=dec, history=hist, terminated=term, windows=windows)


def fixture_path(golden_dir, name):
    return os.path.join(golden_dir, f"behavior_learn_fc_{name}.pt")


def load_fc_case(golden_dir, name):
    """The recorded case with its inputs: args, data {history, terminated}, enc_before / dec_before / enc_after /
    dec_after [A] state dicts, behavior_loss [A], stats, grads0 (agent-net 0's clipped gradients, keys "enc:" / "dec:" +
    name), latent_steps [3] {window, latent}, files {encoder, decoder: [(key, shape)], optimizer: {param id: shape}}."""
    from types import SimpleNamespace
    r = torch.load(fixture_path(golden_dir, name), weights_only=False)
    args = SimpleNamespace(**r["args"])
    x = fc_inputs(name, args)
    enc_after = [{k: v + r["delta_after"][a]["enc:" + k].float() for k, v in x["enc"][a].items()} for a in range(args.n_agents)]
    dec_after = [{k: v + r["delta_after"][a]["dec:" + k].float() for k, v in x["dec"][a].items()} for a in range(args.n_agents)]
    steps = [dict(window=x["windows"][t], latent=out) for t, out in enumerate(r["latent_out"])]
    return dict(args=r["args"], data=dict(history=x["history"], terminated=x["terminated"]), enc_before=x["enc"],
                dec_before=x["dec"], enc_after=enc_after, dec_after=dec_after, behavior_loss=r["behavior_loss"],
                total_loss=r["total_loss"], stability_loss=r["stability_loss"], stats=r["stats"], grads0=r["grads0"],
                latent_steps=steps, files=r["files"])
