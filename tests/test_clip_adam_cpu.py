"""The oracle's clip-plus-Adam step (oracle.iplan_oracle.clip_adam_step), which the GPU tests hold the CUDA learner's
adam_kernel to, against torch.nn.utils.clip_grad_norm_ followed by torch.optim.Adam: gradient norms above and below
max_grad_norm, several steps so that the bias corrections change, float64."""
import copy

import pytest
import torch

from oracle import iplan_oracle as O


@pytest.mark.parametrize("max_norm", [0.05, 10.0])
def test_clip_adam_step_matches_torch(max_norm):
    gen = torch.Generator().manual_seed(7)
    shapes = [(64, 37), (64,), (192, 64), (5, 64), (1,)]
    params = [torch.randn(s, generator=gen, dtype=torch.float64) for s in shapes]
    ref = [torch.nn.Parameter(p.clone()) for p in params]
    opt = torch.optim.Adam(ref, lr=5e-4, eps=1e-5, betas=(0.9, 0.999))
    m = [torch.zeros_like(p) for p in params]
    v = [torch.zeros_like(p) for p in params]
    clipped_steps = 0
    for step in range(1, 8):
        # the gradient norm wanders from about 0.013 to 13, so both sides of max_norm occur for either setting
        scale = 10.0 ** (-4 + (step % 4))
        grads = [torch.randn(s, generator=gen, dtype=torch.float64) * scale for s in shapes]
        for p, g in zip(ref, grads):
            p.grad = g.clone()
        want = torch.nn.utils.clip_grad_norm_(ref, max_norm)
        opt.step()
        got = O.clip_adam_step(params, copy.deepcopy(grads), m, v, step, 5e-4, 1e-5, max_norm)
        clipped_steps += int(float(got) > max_norm)
        assert float(abs(got - want)) <= 1e-14 * float(want)
        st = opt.state
        # torch forms exp_avg with lerp_: agreement to the rounding of the terms, not bit for bit
        close = lambda x, y, g: float((x - y).abs().max()) <= 1e-13 * (float(y.abs().max()) + float(g.abs().max()))
        for p, r, m_, v_, g in zip(params, ref, m, v, grads):
            assert close(m_, st[r]["exp_avg"], 0.1 * g) and close(v_, st[r]["exp_avg_sq"], 1e-3 * g * g)
            assert float((p - r.detach()).abs().max()) <= 1e-15 * float(p.abs().max()) + 1e-12 * 5e-4
    assert 0 < clipped_steps < 7


def test_ppo_epoch_follows_dtype_and_drives_train_agent():
    """ppo_epoch at fixed weights gives train_agent's first-epoch gradients bit for bit, in float64, with its branch
    flags consistent with the per-row quantities it returns."""
    from types import SimpleNamespace
    gen = torch.Generator().manual_seed(3)
    Bf, T, N, o, D, L, A, nA, R = 4, 6, 3, 4, 8, 8, 2, 5, 64
    f64 = torch.float64
    batch = dict(history=torch.rand(Bf, T + 1, N, o, generator=gen, dtype=f64) * 2 - 1,
                 attention_latent=torch.rand(Bf, T + 1, N, D, generator=gen, dtype=f64),
                 behavior_latent=torch.rand(Bf, T + 1, N, L, generator=gen, dtype=f64),
                 actions=torch.randint(0, nA, (Bf, T + 1, 1), generator=gen),
                 available_actions=torch.ones(Bf, T + 1, nA, dtype=f64),
                 reward=torch.randn(Bf, T + 1, 1, generator=gen, dtype=f64) * 20,
                 terminated_masks=torch.ones(Bf, T + 1, 1, dtype=f64),
                 rnn_states_actor=torch.rand(Bf, T + 1, R, generator=gen, dtype=f64),
                 rnn_states_critic=torch.rand(Bf, T + 1, R, generator=gen, dtype=f64))
    batch["actions_onehot"] = torch.nn.functional.one_hot(batch["actions"].squeeze(-1), nA).to(f64)
    obs = O.build_inputs_train(1, batch["history"], batch["attention_latent"], batch["behavior_latent"],
                               batch["actions_onehot"], A)
    assert obs.dtype == f64
    assert torch.equal(obs[..., -A:], torch.tensor([0.0, 1.0], dtype=f64).expand(Bf, T + 1, A))
    Fd = obs.shape[-1]

    def net(kind):
        g = torch.Generator().manual_seed(11 if kind == "actor" else 12)
        keys = O.ACTOR_TRAINABLE if kind == "actor" else O.CRITIC_TRAINABLE
        shapes = {"base.feature_norm.weight": (Fd,), "base.feature_norm.bias": (Fd,), "base.mlp.fc1.0.weight": (64, Fd),
                  "rnn.rnn.weight_ih_l0": (192, 64), "rnn.rnn.weight_hh_l0": (192, 64), "rnn.rnn.bias_ih_l0": (192,),
                  "rnn.rnn.bias_hh_l0": (192,), "base.mlp.fc2.0.0.weight": (64, 64),
                  "act.action_out.linear.weight": (nA, 64), "act.action_out.linear.bias": (nA,),
                  "v_out.weight": (1, 64), "v_out.bias": (1,)}
        return {k: torch.randn(shapes.get(k, (64,)), generator=g, dtype=f64) * (3.0 if "action_out" in k else 0.2)
                for k in keys}

    args = SimpleNamespace(episode_limit=T, batch_size=Bf - 1, n_agents=A, gamma=0.99, gae_lambda=0.95, lr=5e-4,
                           critic_lr=5e-4, optim_eps=1e-5, ppo_epoch=1, clip_param=0.2, entropy_coef=0.01,
                           value_loss_coef=1.0, huber_delta=10.0, max_grad_norm=10.0)
    ap, cp = net("actor"), net("critic")
    perms = [torch.arange((Bf - 1) * T)]
    ap0, cp0 = {k: v.clone() for k, v in ap.items()}, {k: v.clone() for k, v in cp.items()}
    stats, pre, _, _ = O.train_agent(ap, cp, batch, 1, args, perms=perms)
    assert pre["returns"].dtype == f64
    nb = Bf - 1
    alive = batch["terminated_masks"].squeeze(-1)[:nb, :T].reshape(-1)
    flat = dict(obs=obs[:nb, :T].reshape(-1, Fd), rnn_a=batch["rnn_states_actor"][:nb, :T].reshape(nb * T, -1),
                rnn_c=batch["rnn_states_critic"][:nb, :T].reshape(nb * T, -1), act=batch["actions"][:nb, :T].reshape(-1),
                avail=batch["available_actions"][:nb, :T].reshape(nb * T, -1), ret=pre["returns"][:nb].reshape(-1),
                alive=alive, old_lp=pre["old_logp"][:nb].reshape(-1), adv=pre["advantages"][:nb].reshape(-1),
                old_v=pre["values_all"][:nb, :T].reshape(-1))
    e = O.ppo_epoch(ap0, cp0, flat, args, rows_out=True)
    for k, g in stats[0]["grads_actor"].items():
        assert torch.equal(e["grads_actor"][k], g), k
    for k, g in stats[0]["grads_critic"].items():
        assert torch.equal(e["grads_critic"][k], g), k
    assert float(e["actor_grad_norm"]) == stats[0]["actor_grad_norm"]
    assert not any(t.requires_grad for t in list(ap0.values()) + list(cp0.values()))
    # first epoch: ratio 1 and values = old values, so no branch is clipped; the rewards put some rows past the Huber cutoff
    assert not e["ratio_clipped"].any() and not e["value_clip_chosen"].any()
    assert torch.allclose(e["ratio_rows"], torch.ones_like(e["ratio_rows"]), atol=1e-12)
    assert torch.equal(e["huber_dead"], e["e_orig"] < -10.0) and torch.equal(e["huber_outer"], e["e_orig"].abs() > 10.0)
    assert e["d_gi_actor"].shape == (nb * T, 192) and e["a2_critic"].shape == (nb * T, 64)
