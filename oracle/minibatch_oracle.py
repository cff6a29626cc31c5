"""The IPPO update in shuffled mini-batches (num_mini_batch > 1), restated on top of oracle.iplan_oracle.

Reference: IPPOLearner.generate_data (learners/ippo_learner.py:368-424) cuts one permutation of the batch_size * T
training rows per epoch into num_mini_batch index sets of n // num_mini_batch rows (the trailing n % num_mini_batch
rows are not trained on in that epoch); ppo_update (:161-225) takes one clipped Adam step of the actor and one of the
critic per set, with the losses normalised over the set.  Runs in whatever dtype the parameters and the batch carry.
"""
import torch

from . import iplan_oracle as O


def mini_batch_sets(perm, num_mini_batch):
    """generate_data's sampler (:384-386): the index sets of one permutation."""
    mbs = perm.shape[0] // num_mini_batch
    return [perm[m * mbs:(m + 1) * mbs] for m in range(num_mini_batch)]


def ppo_set(actor_p, critic_p, flat, args, idx, alive_sum=None, n_rows=None):
    """Losses and raw gradients of one mini-batch ``idx`` at fixed weights: O.ppo_epoch's result dict.

    ``alive_sum`` / ``n_rows`` replace the set's own sum(alive) and row count as denominators: a rank of a sharded run
    passes the global ones with its share of the set, and the ranks' losses and gradients then add up to the set's.
    A set without an alive row divides by zero in the reference; here its policy and value terms are 0 (no gradient)
    and the entropy bonus, which is not masked, remains."""
    mb = {k: v[idx] for k, v in flat.items()}
    rows = mb["alive"].shape[0]
    asum = mb["alive"].sum() if alive_sum is None else torch.as_tensor(alive_sum, dtype=mb["alive"].dtype)
    n_rows = rows if n_rows is None else n_rows
    if rows and float(asum) > 0 and alive_sum is None:
        return O.ppo_epoch(actor_p, critic_p, mb, args)
    a_tr = [actor_p[k] for k in O.ACTOR_TRAINABLE]
    c_tr = [critic_p[k] for k in O.CRITIC_TRAINABLE]
    zero = torch.zeros((), dtype=mb["alive"].dtype)
    if rows == 0:
        return dict(grads_actor={k: torch.zeros_like(actor_p[k]) for k in O.ACTOR_TRAINABLE},
                    grads_critic={k: torch.zeros_like(critic_p[k]) for k in O.CRITIC_TRAINABLE},
                    policy_loss=zero, value_loss=zero, dist_entropy=zero, ratio=zero)
    inv = 1.0 / asum if float(asum) > 0 else zero
    fresh = [t for t in a_tr + c_tr if not t.requires_grad]
    for t in fresh:
        t.requires_grad_(True)
    try:
        with torch.enable_grad():
            logits, _ = O.actor_logits(actor_p, mb["obs"], mb["rnn_a"], mb["avail"])
            _, lp, ent = O.categorical_stats(logits, mb["act"])
            ent_mean = ent.sum() / n_rows
            values, _ = O.critic_value(critic_p, mb["obs"], mb["rnn_c"])
            ratio = torch.exp(lp - mb["old_lp"])
            surr = torch.min(ratio * mb["adv"], torch.clamp(ratio, 1.0 - args.clip_param, 1.0 + args.clip_param) * mb["adv"])
            pol_loss = (-surr * mb["alive"]).sum() * inv
            g_a = torch.autograd.grad(pol_loss - ent_mean * args.entropy_coef, a_tr)
            v_clip = mb["old_v"] + (values - mb["old_v"]).clamp(-args.clip_param, args.clip_param)
            vl = torch.max(O.huber_one_sided(mb["ret"] - values, args.huber_delta), O.huber_one_sided(mb["ret"] - v_clip, args.huber_delta))
            v_loss = (vl * mb["alive"]).sum() * inv
            g_c = torch.autograd.grad(v_loss * args.value_loss_coef, c_tr, allow_unused=True)
    finally:
        for t in fresh:
            t.requires_grad_(False)
    g_c = [torch.zeros_like(p) if g is None else g for g, p in zip(g_c, c_tr)]
    return dict(grads_actor=dict(zip(O.ACTOR_TRAINABLE, g_a)), grads_critic=dict(zip(O.CRITIC_TRAINABLE, g_c)),
                policy_loss=pol_loss.detach(), value_loss=v_loss.detach(), dist_entropy=ent_mean.detach(),
                ratio=ratio.detach().sum() / n_rows)


def agent_rows(actor_p, critic_p, batch, agent_id, args):
    """The per-row tensors of one agent's training rows r = b * T + t (all stored episodes; the permutations index the
    first batch_size * T), with the pre-update returns, normalised advantages, old log-probs and old values computed
    once, as O.train_agent computes them (learners/ippo_learner.py:254-282)."""
    T = args.episode_limit
    obs_all = O.build_inputs_train(agent_id, batch["history"], batch["attention_latent"], batch["behavior_latent"],
                                   batch["actions_onehot"], args.n_agents)
    Bf, Fd = obs_all.shape[0], obs_all.shape[-1]
    alive_all = batch["terminated_masks"].squeeze(-1).to(obs_all.dtype)
    rnn_c_all = batch["rnn_states_critic"]
    flat2 = lambda x: x[:, :T].reshape(Bf * T, -1)
    with torch.no_grad():
        v_all, _ = O.critic_value(critic_p, obs_all.reshape(-1, Fd), rnn_c_all.reshape(-1, rnn_c_all.shape[-1]))
        v_all = v_all.view(Bf, T + 1)
        returns = O.gae_returns(v_all, batch["reward"][:, :-1].squeeze(-1), alive_all, args.gamma, args.gae_lambda)
        adv = O.normalised_advantages(returns, v_all[:, :T], alive_all[:, :T])
        logits, _ = O.actor_logits(actor_p, flat2(obs_all), flat2(batch["rnn_states_actor"]), flat2(batch["available_actions"]))
        _, old_lp, _ = O.categorical_stats(logits, batch["actions"][:, :T].reshape(-1))
    return dict(obs=flat2(obs_all), rnn_a=flat2(batch["rnn_states_actor"]), rnn_c=flat2(rnn_c_all),
                act=batch["actions"][:, :T].reshape(-1), avail=flat2(batch["available_actions"]), ret=returns.reshape(-1),
                alive=alive_all[:, :T].reshape(-1), old_lp=old_lp, adv=adv.reshape(-1), old_v=v_all[:, :T].reshape(-1))


def train_agent(actor_p, critic_p, batch, agent_id, args, perms, num_mini_batch, opt_a=None, opt_c=None):
    """One agent's share of IPPOLearner.train with ``num_mini_batch`` sets per epoch; ``perms[epoch]`` is the epoch's
    permutation of the batch_size * T training rows.  Updates the parameters in place; returns one statistics dict per
    Adam step (ppo_epoch * num_mini_batch of them) and the optimiser states."""
    flat = agent_rows(actor_p, critic_p, batch, agent_id, args)
    a_tr = [actor_p[k] for k in O.ACTOR_TRAINABLE]
    c_tr = [critic_p[k] for k in O.CRITIC_TRAINABLE]
    opt_a = opt_a or O.AdamState(a_tr, args.lr, args.optim_eps)
    opt_c = opt_c or O.AdamState(c_tr, args.critic_lr, args.optim_eps)
    stats = []
    for ep in range(args.ppo_epoch):
        for idx in mini_batch_sets(torch.as_tensor(perms[ep]).long(), num_mini_batch):
            e = ppo_set(actor_p, critic_p, flat, args, idx)
            with torch.no_grad():
                n_a = opt_a.clip_step([e["grads_actor"][k] for k in O.ACTOR_TRAINABLE], args.max_grad_norm)
                n_c = opt_c.clip_step([e["grads_critic"][k] for k in O.CRITIC_TRAINABLE], args.max_grad_norm)
            stats.append(dict(value_loss=float(e["value_loss"]), policy_loss=float(e["policy_loss"]),
                              dist_entropy=float(e["dist_entropy"]), actor_grad_norm=float(n_a),
                              critic_grad_norm=float(n_c), ratio=float(e["ratio"])))
    return stats, opt_a, opt_c


def agent_batch(data, a, n_actions, dtype=torch.float32):
    """Agent a's SeparatedReplayBuffer.get_batch() view of EpisodeBatch-shaped ``data`` [B, T+1, A, ...]."""
    f = lambda k: torch.as_tensor(data[k])[:, :, a].to(dtype)
    acts = torch.as_tensor(data["actions"])[:, :, a].long()
    return dict(history=f("history"), attention_latent=f("attention_latent"), behavior_latent=f("behavior_latent"),
                actions=acts, actions_onehot=torch.nn.functional.one_hot(acts.squeeze(-1), n_actions).to(dtype),
                available_actions=torch.as_tensor(data["avail_actions"])[:, :, a], reward=f("reward"),
                terminated_masks=1 - f("terminated"), rnn_states_actor=f("rnn_states_actors"),
                rnn_states_critic=f("rnn_states_critics"))
