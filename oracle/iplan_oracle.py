"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

CPU restatement (PyTorch fp32 on the host cores) of the reference's iPLAN hot
path.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this module, and only as
the checker or the timed CPU baseline; nothing under ``iplan_b200/`` imports it.

Pinning: the reference ships no tests or golden vectors for this path
(SURVEY.md §4), so the oracle is pinned against outputs of the reference's own
modules executed in the build container: ``tests/golden/make_golden.py`` imports
``/root/reference`` and writes ``tests/golden/*.pt``; ``tests/test_oracle_golden.py``
checks every function below against those fixtures (<=2e-6 abs).

Every function cites the reference lines it restates.  Weights are passed as
``dict[str, Tensor]`` using the reference modules' ``state_dict`` key names.
"""
import math

import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------
# shared pieces
# ----------------------------------------------------------------------------------

def neighbour_index(n):
    """[n, n-1] table j(i, s) = s if s < i else s + 1  (nova/GAT_Net.py:61-66, :111-113)."""
    i = torch.arange(n).view(n, 1)
    s = torch.arange(n - 1).view(1, n - 1)
    return torch.where(s < i, s, s + 1)


def gru_cell(x_proj, h, w_hh, b_hh):
    """One GRU step given the already-projected input ``x_proj = W_ih x + b_ih``.
    PyTorch gate order r, z, n;  n = tanh(i_n + r * (W_hn h + b_hn));
    h' = (1 - z) * n + z * h   (torch.nn.GRU / GRUCell semantics used at
    nova/GAT_Net.py:26,39, nova/behavior_net.py:14, utils/mappo_utils/rnn.py:13)."""
    hd = h.shape[-1]
    gh = h @ w_hh.t() + b_hh
    r = torch.sigmoid(x_proj[..., :hd] + gh[..., :hd])
    z = torch.sigmoid(x_proj[..., hd:2 * hd] + gh[..., hd:2 * hd])
    n = torch.tanh(x_proj[..., 2 * hd:] + r * gh[..., 2 * hd:])
    return (1.0 - z) * n + z * h


def gumbel_from_exponential(e):
    """F.gumbel_softmax draws ``-empty_like(logits).exponential_().log()``
    (torch/nn/functional.py); the reference calls it at nova/GAT_Net.py:93."""
    return -e.log()


def draw_gumbel(rows, generator=None):
    """Noise with the reference's draw order: one [rows, 2] exponential tensor per
    GAT_Net.forward call, rows ordered ((b*N + i)*(N-1) + s)  (nova/GAT_Net.py:85-93)."""
    e = torch.empty(rows, 2).exponential_(generator=generator)
    return gumbel_from_exponential(e)


# ----------------------------------------------------------------------------------
# a2  GAT_Net.forward  (nova/GAT_Net.py:41-142)
# ----------------------------------------------------------------------------------

def gat_forward(p, obs, h_prev, gumbel, tau=0.01, return_parts=False):
    """obs [B, N, in], h_prev [B*N, D], gumbel [B, N, N-1, 2] -> new hidden [B*N, D].

    Vectorised restatement; uses the factorised input projection
    W_ih [h_i; h_j] = W_ih[:, :H] h_i + W_ih[:, H:] h_j  (SURVEY Appendix A)."""
    B, N, _ = obs.shape
    H = p["encoding.weight"].shape[0]
    D = p["q.weight"].shape[0]
    enc = F.relu(obs @ p["encoding.weight"].t() + p["encoding.bias"])            # :50
    idx = neighbour_index(N)                                                     # [N, N-1]

    outs = []
    for sfx, order in (("", range(N - 1)), ("_reverse", range(N - 2, -1, -1))):  # :26, :83
        w_ih = p["hard_bi_GRU.weight_ih_l0" + sfx]
        w_hh = p["hard_bi_GRU.weight_hh_l0" + sfx]
        b_ih = p["hard_bi_GRU.bias_ih_l0" + sfx]
        b_hh = p["hard_bi_GRU.bias_hh_l0" + sfx]
        ego = enc @ w_ih[:, :H].t() + b_ih                                       # [B, N, 3H]
        nbr = enc @ w_ih[:, H:].t()                                              # [B, N, 3H]
        h = torch.zeros(B, N, H, dtype=obs.dtype)                                # :78
        out = torch.empty(B, N, N - 1, H, dtype=obs.dtype)
        for s in order:
            gi = ego + nbr[:, idx[:, s], :]
            h = gru_cell(gi, h, w_hh, b_hh)
            out[:, :, s] = h
        outs.append(out)
    hh = torch.cat(outs, dim=-1)                                                 # [B,N,N-1,2H]
    logits = hh @ p["hard_encoding.weight"].t() + p["hard_encoding.bias"]        # :91
    hard = torch.softmax((logits + gumbel) / tau, dim=-1)[..., 1]                # :93-95

    h_out = enc.reshape(-1, H)
    q = (h_out @ p["q.weight"].t()).view(B, N, D)                                # :101
    k = (h_out @ p["k.weight"].t()).view(B, N, D)                                # :103
    v = F.relu(h_out @ p["v.weight"].t() + p["v.bias"]).view(B, N, D)            # :105
    score = torch.einsum("bid,bjd->bij", q, k) / float(math.sqrt(D))             # :123-126
    score = torch.gather(score, 2, idx.unsqueeze(0).expand(B, -1, -1))           # drop j == i
    soft = torch.softmax(score, dim=-1)                                          # :129
    w = soft * hard                                                              # :132 (no renorm)
    x = torch.einsum("bis,bisd->bid", w, v[:, idx, :])                           # [B, N, D]
    x = x.reshape(-1, D)
    gi = x @ p["rnn.weight_ih"].t() + p["rnn.bias_ih"]                           # :140 GRUCell
    new_h = gru_cell(gi, h_prev, p["rnn.weight_hh"], p["rnn.bias_hh"])
    if return_parts:
        return new_h, dict(enc=enc, logits=logits, hard=hard, soft=soft, x=x)
    return new_h


def gat_forward_loops(p, obs, h_prev, gumbel, tau=0.01):
    """Same result as ``gat_forward`` but executing the op sequence the reference
    executes on the CPU (per-ego Python loops that cat/stack [h_i, h_j] pairs, one
    bidirectional nn.GRU over the N-1 axis, per-ego attention loop:
    nova/GAT_Net.py:57-75, :83, :107-133).  Used only as the timed CPU baseline,
    because that op sequence — not the arithmetic — is where the reference spends
    its time (SURVEY §3.2)."""
    B, N, _ = obs.shape
    H = p["encoding.weight"].shape[0]
    D = p["q.weight"].shape[0]
    enc = F.relu(F.linear(obs, p["encoding.weight"], p["encoding.bias"]))
    pair_seqs = []
    for i in range(N):
        ego = enc[:, i]
        pairs = [torch.cat([ego, enc[:, j]], dim=-1) for j in range(N) if j != i]
        pair_seqs.append(torch.stack(pairs, dim=0))
    seq = torch.stack(pair_seqs, dim=-2).view(N - 1, -1, 2 * H)
    flat = [p["hard_bi_GRU.weight_ih_l0"], p["hard_bi_GRU.weight_hh_l0"],
            p["hard_bi_GRU.bias_ih_l0"], p["hard_bi_GRU.bias_hh_l0"],
            p["hard_bi_GRU.weight_ih_l0_reverse"], p["hard_bi_GRU.weight_hh_l0_reverse"],
            p["hard_bi_GRU.bias_ih_l0_reverse"], p["hard_bi_GRU.bias_hh_l0_reverse"]]
    h0 = torch.zeros(2, B * N, H)
    hh, _ = torch._VF.gru(seq, h0, flat, True, 1, 0.0, False, True, False)
    hh = hh.permute(1, 0, 2).reshape(-1, 2 * H)
    logits = F.linear(hh, p["hard_encoding.weight"], p["hard_encoding.bias"])
    hard = torch.softmax((logits + gumbel.reshape(-1, 2)) / tau, dim=-1)[:, 1]
    hard = hard.view(-1, N, 1, N - 1).permute(1, 0, 2, 3)
    flat_enc = enc.reshape(-1, H)
    q = F.linear(flat_enc, p["q.weight"]).reshape(-1, N, D)
    k = F.linear(flat_enc, p["k.weight"]).reshape(-1, N, D)
    v = F.relu(F.linear(flat_enc, p["v.weight"], p["v.bias"])).reshape(-1, N, D)
    xs = []
    for i in range(N):
        q_i = q[:, i].view(-1, 1, D)
        k_i = torch.stack([k[:, j] for j in range(N) if j != i], dim=0).permute(1, 2, 0)
        v_i = torch.stack([v[:, j] for j in range(N) if j != i], dim=0).permute(1, 2, 0)
        soft = torch.softmax(torch.matmul(q_i, k_i) / float(math.sqrt(D)), dim=-1)
        xs.append((v_i * soft * hard[i]).sum(dim=-1))
    x = torch.stack(xs, dim=1).reshape(-1, D)
    gi = F.linear(x, p["rnn.weight_ih"], p["rnn.bias_ih"])
    return gru_cell(gi, h_prev, p["rnn.weight_hh"], p["rnn.bias_hh"])


def gat_latent_update(gat_params, history_single, encoder_hidden, behavior_latent, gumbel,
                      loops=False, dtype=torch.float32):
    """a1  Prediction_policy.GAT_latent_update (nova/prediction_policy.py:92-118).
    history_single [B,A,N,o], encoder_hidden [B,A,N,D], behavior_latent [B,A,N,L],
    gumbel [A,B,N,N-1,2] -> [B,A,N,D], computed in ``dtype`` (the parameters must have it too)."""
    hs = torch.as_tensor(history_single, dtype=dtype)
    eh = torch.as_tensor(encoder_hidden, dtype=dtype)
    bl = torch.as_tensor(behavior_latent, dtype=dtype)
    gumbel = torch.as_tensor(gumbel, dtype=dtype)
    B, A, N, _ = hs.shape
    D = eh.shape[-1]
    fn = gat_forward_loops if loops else gat_forward
    outs = []
    for a in range(A):
        x = torch.cat([hs[:, a], bl[:, a]], dim=-1)                              # :104-105
        h = eh[:, a].reshape(B * N, D)                                           # :107-108
        outs.append(fn(gat_params[a], x, h, gumbel[a]).view(B, 1, N, D))         # :110-113
    return torch.cat(outs, dim=1)


# ----------------------------------------------------------------------------------
# a3  EncoderRNN.forward + Behavior_policy.latent_update
# ----------------------------------------------------------------------------------

def behavior_encoder(p, window, hidden):
    """nova/behavior_net.py:17-22.  window [M, W, o], hidden [M, E] ->
    (new hidden [M, E], latent [M, L])."""
    u = F.relu(window @ p["linear.weight"].t() + p["linear.bias"])
    h = hidden
    for t in range(window.shape[1]):
        gi = u[:, t] @ p["rnn.weight_ih_l0"].t() + p["rnn.bias_ih_l0"]
        h = gru_cell(gi, h, p["rnn.weight_hh_l0"], p["rnn.bias_hh_l0"])
    latent = torch.softmax(h @ p["out.weight"].t() + p["out.bias"], dim=-1)
    return h, latent


def behavior_latent_update(enc_params, history, encoder_hidden, prev_latent, coef=0.1):
    """nova/stable_behavior_policy.py:83-123.  history [B,A,N,W,o],
    encoder_hidden [B,1,A,N,E], prev_latent [B,A,N,L] ->
    (new latent [B,A,N,L] = (1-coef)*prev + coef*latent, new hidden [B,1,A,N,E])."""
    hist = torch.as_tensor(history, dtype=torch.float32)
    hid = torch.as_tensor(encoder_hidden, dtype=torch.float32)
    prev = torch.as_tensor(prev_latent, dtype=torch.float32)
    B, A, N, W, o = hist.shape
    E = hid.shape[-1]
    lat, newh = [], []
    for a in range(A):
        h, z = behavior_encoder(enc_params[a], hist[:, a].reshape(B * N, W, o),
                                hid[:, 0, a].reshape(B * N, E))
        lat.append(z.view(B, 1, N, -1))
        newh.append(h.view(B, 1, 1, N, E))
    new_latent = torch.cat(lat, dim=1)
    new_latent = (1 - coef) * prev + new_latent * coef                           # :118
    return new_latent, torch.cat(newh, dim=2)


# ----------------------------------------------------------------------------------
# a4-a7  controller: input assembly, actor, critic
# ----------------------------------------------------------------------------------

def build_inputs_step(history, attention, behavior, last_onehot, n_agents):
    """DcntrlMAC._build_inputs (controllers/dcntrl_controller.py:187-213) for one
    timestep.  history [B,A,N,o], attention [B,A,N,D], behavior [B,A,N,L],
    last_onehot [B,A,n_act] (zeros at t == 0) -> [B, A, F]."""
    B = history.shape[0]
    slots = torch.cat([history, attention, behavior], dim=-1).reshape(B, n_agents, -1)
    eye = torch.eye(n_agents).unsqueeze(0).expand(B, -1, -1)
    return torch.cat([slots, last_onehot.reshape(B, n_agents, -1), eye], dim=2)


def build_inputs_train(agent_id, history, attention, behavior, actions_onehot, n_agents):
    """DcntrlMAC._build_inputs_ippo (:87-115) for one agent, all timesteps.
    history [Bf,T+1,N,o] ..., actions_onehot [Bf,T+1,n_act] -> [Bf, T+1, F].
    Quirk kept: the "last action" at t = 0 is the action taken AT t = 0 (:107)."""
    bs, ts = history.shape[:2]
    slots = torch.cat([history, attention, behavior], dim=-1).reshape(bs, ts, -1)
    last = torch.cat([actions_onehot[:, 0:1], actions_onehot[:, :-1]], dim=1)
    ident = torch.zeros(bs, ts, n_agents, dtype=history.dtype, device=history.device)
    ident[:, :, agent_id] = 1
    return torch.cat([slots, last, ident], dim=-1)


def trunk_forward(p, obs, h0, taps=None):
    """MLPBase + RNNLayer (utils/mappo_utils/mlp.py:50-56, :24-28; rnn.py:24-78) for
    rows of length-1 sequences: obs [R, F], h0 [R, Rh] -> (features [R, Rh], h1 [R, Rh]).
    ``fc_h`` exists in the state_dict but is never called (mlp.py:20-27).
    ``taps`` (a dict) receives the GRU input ``a2`` [R, Rh], its projection ``gi`` [R, 3 Rh] and the two ReLUs'
    inputs ``z1`` / ``z2`` and outputs ``r1`` / ``r2``."""
    x = F.layer_norm(obs, obs.shape[-1:], p["base.feature_norm.weight"],
                     p["base.feature_norm.bias"], 1e-5)
    z1 = x @ p["base.mlp.fc1.0.weight"].t() + p["base.mlp.fc1.0.bias"]
    r1 = F.relu(z1)
    x = F.layer_norm(r1, r1.shape[-1:], p["base.mlp.fc1.2.weight"], p["base.mlp.fc1.2.bias"], 1e-5)
    z2 = x @ p["base.mlp.fc2.0.0.weight"].t() + p["base.mlp.fc2.0.0.bias"]
    r2 = F.relu(z2)
    x = F.layer_norm(r2, r2.shape[-1:], p["base.mlp.fc2.0.2.weight"], p["base.mlp.fc2.0.2.bias"], 1e-5)
    gi = x @ p["rnn.rnn.weight_ih_l0"].t() + p["rnn.rnn.bias_ih_l0"]
    if taps is not None:
        taps.update(a2=x, gi=gi, z1=z1, r1=r1, z2=z2, r2=r2)
    h1 = gru_cell(gi, h0, p["rnn.rnn.weight_hh_l0"], p["rnn.rnn.bias_hh_l0"])
    feat = F.layer_norm(h1, h1.shape[-1:], p["rnn.norm.weight"], p["rnn.norm.bias"], 1e-5)
    return feat, h1


def actor_logits(p, obs, h0, avail=None, taps=None):
    """R_Actor trunk + Categorical head (modules/agents/ippo_actor.py:43-72,
    utils/mappo_utils/distributions.py:64-68): masked logits [R, n_act], h1."""
    feat, h1 = trunk_forward(p, obs, h0, taps)
    logits = feat @ p["act.action_out.linear.weight"].t() + p["act.action_out.linear.bias"]
    if avail is not None:
        logits = torch.where(avail == 0, torch.full_like(logits, -1e10), logits)
    return logits, h1


def categorical_stats(logits, actions=None):
    """torch.distributions.Categorical(logits=...) quantities used by
    FixedCategorical (distributions.py:14-28): normalised log-probs, log_prob of
    ``actions`` [R] and entropy [R]."""
    logp_all = logits - logits.logsumexp(dim=-1, keepdim=True)
    probs = logp_all.exp()
    min_real = torch.finfo(logp_all.dtype).min
    ent = -(torch.clamp(logp_all, min=min_real) * probs).sum(-1)
    lp = None
    if actions is not None:
        lp = logp_all.gather(-1, actions.long().view(-1, 1)).squeeze(-1)
    return logp_all, lp, ent


def critic_value(p, obs, h0, taps=None):
    """R_Critic.forward (modules/critics/ippo_critic.py:47-65); PopArt is a plain
    Linear here (utils/mappo_utils/popart.py:41-46)."""
    feat, h1 = trunk_forward(p, obs, h0, taps)
    v = feat @ p["v_out.weight"].t() + p["v_out.bias"]
    return v.squeeze(-1), h1


def inverse_cdf(probs, u):
    """Categorical sampling by inverse CDF: probs [R, n_act], u [R] -> the first action whose cdf exceeds u.  Like
    torch.distributions.Categorical it never returns a zero-probability action: where u is at or above the last cdf
    (u = 1, or the sum of the probabilities falls short of 1) it returns the last action with probability > 0."""
    n = probs.shape[-1]
    act = (u.view(-1, 1).to(probs.dtype) >= probs.cumsum(-1)).sum(-1).clamp(max=n - 1)
    pos = torch.arange(n).expand_as(probs)
    cand = torch.where((probs > 0) & (pos <= act.view(-1, 1)), pos, torch.full_like(pos, -1)).amax(-1)
    first = torch.where(probs > 0, pos, torch.full_like(pos, n)).amin(-1)
    return torch.where(cand >= 0, cand, first)


def select_actions(actor_params, critic_params, inputs, avail, rnn_a, rnn_c,
                   test_mode=False, uniforms=None):
    """a5  DcntrlMAC.select_actions_ippo (controllers/dcntrl_controller.py:27-58) with
    the sampling noise made explicit: ``uniforms`` [B, A] in [0,1) select the action by
    inverse CDF over the probabilities (the reference samples with torch.multinomial;
    parity tests compare logits / log-probs / values / hidden states and use
    test_mode=True for the argmax path).  inputs [B,A,F], avail [B,A,n_act],
    rnn_* [B,A,R] -> dict."""
    B, A, _ = inputs.shape
    out = dict(values=[], actions=[], logp=[], rnn_a=[], rnn_c=[], logits=[])
    for a in range(A):
        logits, h1 = actor_logits(actor_params[a], inputs[:, a], rnn_a[:, a], avail[:, a])
        logp_all, _, _ = categorical_stats(logits)
        probs = logp_all.exp()
        if test_mode or uniforms is None:
            act = probs.argmax(dim=-1)                                           # mode()
        else:
            act = inverse_cdf(probs, uniforms[:, a])
        out["logits"].append(logits)
        out["actions"].append(act)
        out["logp"].append(logp_all.gather(-1, act.view(-1, 1)).squeeze(-1))
        out["rnn_a"].append(h1)
        v, hc = critic_value(critic_params[a], inputs[:, a], rnn_c[:, a])
        out["values"].append(v)
        out["rnn_c"].append(hc)
    return {k: torch.stack(v, dim=1) for k, v in out.items()}


# ----------------------------------------------------------------------------------
# a11-a16  learner
# ----------------------------------------------------------------------------------

def gae_returns(values_all, rewards, alive_all, gamma=0.99, lam=0.95):
    """IPPOLearner.compute_returns (learners/ippo_learner.py:344-365), GAE branch.
    values_all [Bf,T+1], rewards [Bf,T], alive_all [Bf,T+1] -> returns [Bf,T]."""
    T = rewards.shape[1]
    ret = torch.empty_like(rewards)
    gae = torch.zeros(rewards.shape[0], dtype=rewards.dtype, device=rewards.device)
    for t in reversed(range(T)):
        delta = rewards[:, t] + gamma * values_all[:, t + 1] * alive_all[:, t + 1] - values_all[:, t]
        gae = delta + gamma * lam * alive_all[:, t + 1] * gae
        ret[:, t] = gae + values_all[:, t]
    return ret


def normalised_advantages(returns, values, alive):
    """learners/ippo_learner.py:272-279: zero where the agent is not alive, then
    (x - mean) / (std + 1e-5) with the UNBIASED std over every entry incl. the zeros."""
    adv = (returns - values).clone()
    adv[alive == 0.0] = 0.0
    std, mean = torch.std_mean(adv)
    return (adv - mean) / (std + 1e-5)


def huber_one_sided(e, d):
    """utils/mappo_utils/util.py:33-36 — as written: e < -d contributes 0."""
    a = (e.abs() <= d).float()
    b = (e > d).float()
    return a * e ** 2 / 2 + b * d * (e.abs() - d / 2)


def policy_loss_terms(logp, old_logp, adv, alive, clip=0.2):
    """learners/ippo_learner.py:185-197."""
    ratio = torch.exp(logp - old_logp)
    surr1 = ratio * adv
    surr2 = torch.clamp(ratio, 1.0 - clip, 1.0 + clip) * adv
    loss = (-torch.min(surr1, surr2) * alive).sum() / alive.sum()
    return loss, ratio


def value_loss_terms(values, old_values, returns, alive, clip=0.2, delta=10.0):
    """IPPOLearner.cal_value_loss (learners/ippo_learner.py:128-159), huber + clipped
    + active masks."""
    v_clip = old_values + (values - old_values).clamp(-clip, clip)
    l_clip = huber_one_sided(returns - v_clip, delta)
    l_orig = huber_one_sided(returns - values, delta)
    loss = torch.max(l_orig, l_clip)
    return (loss * alive).sum() / alive.sum()


ACTOR_TRAINABLE = [
    "base.feature_norm.weight", "base.feature_norm.bias",
    "base.mlp.fc1.0.weight", "base.mlp.fc1.0.bias", "base.mlp.fc1.2.weight", "base.mlp.fc1.2.bias",
    "base.mlp.fc2.0.0.weight", "base.mlp.fc2.0.0.bias", "base.mlp.fc2.0.2.weight", "base.mlp.fc2.0.2.bias",
    "rnn.rnn.weight_ih_l0", "rnn.rnn.weight_hh_l0", "rnn.rnn.bias_ih_l0", "rnn.rnn.bias_hh_l0",
    "rnn.norm.weight", "rnn.norm.bias",
    "act.action_out.linear.weight", "act.action_out.linear.bias",
]
CRITIC_TRAINABLE = ACTOR_TRAINABLE[:-2] + ["v_out.weight", "v_out.bias"]


class AdamState:
    """torch.optim.Adam(lr, eps, betas=(0.9, 0.999), wd=0) restated on a list of
    tensors (learners/ippo_learner.py:74-81); bias correction as torch does it:
    step_size = lr / (1 - b1^t); denom = sqrt(v) / sqrt(1 - b2^t) + eps."""

    def __init__(self, params, lr, eps, b1=0.9, b2=0.999):
        self.params, self.lr, self.eps, self.b1, self.b2 = params, lr, eps, b1, b2
        self.m = [torch.zeros_like(p) for p in params]
        self.v = [torch.zeros_like(p) for p in params]
        self.t = 0

    def step(self, grads):
        self.t += 1
        adam_update(self.params, grads, self.m, self.v, self.t, self.lr, self.eps, self.b1, self.b2)

    def clip_step(self, grads, max_norm):
        """clip_grad_norm_(max_norm) and then ``step``; returns the norm before clipping."""
        self.t += 1
        return clip_adam_step(self.params, grads, self.m, self.v, self.t, self.lr, self.eps, max_norm, self.b1, self.b2)


def adam_update(params, grads, m, v, step, lr, eps, b1=0.9, b2=0.999):
    """Adam step number ``step`` (1-based) on lists of tensors, in place: torch.optim.Adam's arithmetic (see AdamState)."""
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    for p_, g, m_, v_ in zip(params, grads, m, v):
        m_.mul_(b1).add_(g, alpha=1 - b1)
        v_.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (v_.sqrt() / math.sqrt(bc2)).add_(eps)
        p_.addcdiv_(m_, denom, value=-lr / bc1)


def clip_grads(grads, max_norm):
    """nn.utils.clip_grad_norm_ (learners/ippo_learner.py:205, :219): total 2-norm,
    scale by max_norm / (norm + 1e-6) clamped to 1."""
    total = torch.sqrt(sum((g.detach() ** 2).sum() for g in grads))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return [g * coef for g in grads], total


def clip_adam_step(params, grads, m, v, step, lr, eps, max_norm, b1=0.9, b2=0.999):
    """One optimiser step of the IPPO update (learners/ippo_learner.py:205-221): clip_grad_norm_(max_norm) of the raw
    gradients, then Adam step ``step``; params / m / v are updated in place, in their own dtype.  Returns the norm
    before clipping."""
    clipped, total = clip_grads(grads, max_norm)
    adam_update(params, clipped, m, v, step, lr, eps, b1, b2)
    return total


def ppo_epoch(actor_p, critic_p, flat, args, idx=None, rows_out=False):
    """One PPO epoch of IPPOLearner.train (learners/ippo_learner.py:181-221) at fixed weights, up to the raw gradients.

    ``flat`` holds the per-row tensors of the trained episodes (obs, rnn_a, rnn_c, act, avail, and the pre-update ret,
    alive, old_lp, adv (normalised), old_v); ``idx`` is the epoch's row order (None: as stored).  Returns a dict: the
    raw gradients ``grads_actor`` / ``grads_critic`` (keyed like ACTOR_TRAINABLE / CRITIC_TRAINABLE), the 0-d tensors
    ``policy_loss``, ``value_loss``, ``dist_entropy``, ``ratio`` (mean), ``actor_grad_norm``, ``critic_grad_norm``.
    ``rows_out`` adds, per row in that order: ``logp``, ``value``, ``entropy``, ``ratio_rows``, the value errors
    ``e_orig`` = ret - v and ``e_clip`` = ret - v_clipped with their losses ``l_orig`` / ``l_clip``; the branch flags
    ``ratio_clipped`` (the clipped surrogate is the minimum: no policy gradient), ``value_clip_chosen`` (the clipped
    value loss is the maximum), ``huber_outer`` (|e| > delta for the chosen e) and ``huber_dead`` (e < -delta: no
    gradient); the GRU inputs ``a2_actor`` / ``a2_critic`` and the loss gradients w.r.t. their projections
    ``d_gi_actor`` / ``d_gi_critic``; the two ReLUs' inputs ``z_actor`` / ``z_critic`` (z1, z2) and the loss gradients
    w.r.t. their outputs ``d_relu_actor`` / ``d_relu_critic``."""
    mb = flat if idx is None else {k: v[idx] for k, v in flat.items()}
    a_tr = [actor_p[k] for k in ACTOR_TRAINABLE]
    c_tr = [critic_p[k] for k in CRITIC_TRAINABLE]
    fresh = [t for t in a_tr + c_tr if not t.requires_grad]
    for t in fresh:
        t.requires_grad_(True)
    tap_a, tap_c = ({}, {}) if rows_out else (None, None)
    try:
        with torch.enable_grad():
            logits, _ = actor_logits(actor_p, mb["obs"], mb["rnn_a"], mb["avail"], taps=tap_a)
            _, lp, ent = categorical_stats(logits, mb["act"])
            ent_mean = ent.mean()                                                    # act.py:164 (unmasked)
            values, _ = critic_value(critic_p, mb["obs"], mb["rnn_c"], taps=tap_c)
            pol_loss, ratio = policy_loss_terms(lp, mb["old_lp"], mb["adv"], mb["alive"], args.clip_param)
            extra_a = [tap_a["gi"], tap_a["r1"], tap_a["r2"]] if rows_out else []
            g_a = torch.autograd.grad(pol_loss - ent_mean * args.entropy_coef, a_tr + extra_a)
            v_loss = value_loss_terms(values, mb["old_v"], mb["ret"], mb["alive"], args.clip_param, args.huber_delta)
            extra_c = [tap_c["gi"], tap_c["r1"], tap_c["r2"]] if rows_out else []
            g_c = torch.autograd.grad(v_loss * args.value_loss_coef, c_tr + extra_c)
    finally:
        for t in fresh:
            t.requires_grad_(False)
    raw_a, raw_c = list(g_a[:len(a_tr)]), list(g_c[:len(c_tr)])
    norm = lambda gs: torch.sqrt(sum((g.detach() ** 2).sum() for g in gs))         # clip_grads' total
    out = dict(grads_actor=dict(zip(ACTOR_TRAINABLE, raw_a)), grads_critic=dict(zip(CRITIC_TRAINABLE, raw_c)),
               policy_loss=pol_loss.detach(), value_loss=v_loss.detach(), dist_entropy=ent_mean.detach(),
               ratio=ratio.mean().detach(), actor_grad_norm=norm(raw_a), critic_grad_norm=norm(raw_c))
    if rows_out:
        with torch.no_grad():
            clip, d = args.clip_param, args.huber_delta
            v = values.detach()
            v_clip = mb["old_v"] + (v - mb["old_v"]).clamp(-clip, clip)
            e_orig, e_clip = mb["ret"] - v, mb["ret"] - v_clip
            l_orig, l_clip = huber_one_sided(e_orig, d), huber_one_sided(e_clip, d)
            r = ratio.detach()
            chosen = l_clip > l_orig
            e = torch.where(chosen, e_clip, e_orig)
            out.update(logp=lp.detach(), value=v, entropy=ent.detach(), ratio_rows=r, e_orig=e_orig, e_clip=e_clip,
                       l_orig=l_orig, l_clip=l_clip, ratio_clipped=r.clamp(1 - clip, 1 + clip) * mb["adv"] < r * mb["adv"],
                       value_clip_chosen=chosen, huber_outer=e.abs() > d, huber_dead=e < -d,
                       a2_actor=tap_a["a2"].detach(), a2_critic=tap_c["a2"].detach(), d_gi_actor=g_a[-3], d_gi_critic=g_c[-3],
                       z_actor=(tap_a["z1"].detach(), tap_a["z2"].detach()), z_critic=(tap_c["z1"].detach(), tap_c["z2"].detach()),
                       d_relu_actor=tuple(g_a[-2:]), d_relu_critic=tuple(g_c[-2:]))
    return out


def train_agent(actor_p, critic_p, batch, agent_id, args, opt_a=None, opt_c=None,
                perms=None):
    """One agent's share of IPPOLearner.train (learners/ippo_learner.py:249-312).

    ``batch`` holds the per-agent SeparatedReplayBuffer.get_batch() tensors
    (utils/mappo_utils/separated_buffer.py:71-94): history [Bf,T+1,N,o],
    attention_latent, behavior_latent, actions [Bf,T+1,1] (long), actions_onehot,
    available_actions, reward [Bf,T+1,1], terminated_masks [Bf,T+1,1] (alive = 1),
    rnn_states_actor / rnn_states_critic [Bf,T+1,R].
    Updates ``actor_p`` / ``critic_p`` in place; returns per-update stats and the
    pre-update tensors (returns, advantages, old log-probs, values)."""
    T = args.episode_limit
    nb = args.batch_size                      # episodes actually trained on (:371)
    rows = nb * T
    obs_all = build_inputs_train(agent_id, batch["history"], batch["attention_latent"],
                                 batch["behavior_latent"], batch["actions_onehot"], args.n_agents)
    Bf = obs_all.shape[0]
    Fdim = obs_all.shape[-1]
    alive_all = batch["terminated_masks"].squeeze(-1).float()
    rewards = batch["reward"][:, :-1].squeeze(-1)
    actions = batch["actions"][:, :-1].squeeze(-1)
    avail = batch["available_actions"][:, :-1]
    rnn_a = batch["rnn_states_actor"][:, :-1]
    rnn_c_all = batch["rnn_states_critic"]

    with torch.no_grad():
        v_all, _ = critic_value(critic_p, obs_all.reshape(-1, Fdim), rnn_c_all.reshape(-1, rnn_c_all.shape[-1]))
        v_all = v_all.view(Bf, T + 1)
        returns = gae_returns(v_all, rewards, alive_all, args.gamma, args.gae_lambda)
        cur_v = v_all[:, :T]
        alive = alive_all[:, :T]
        adv = normalised_advantages(returns, cur_v, alive)
        obs = obs_all[:, :T].reshape(-1, Fdim)
        logits, _ = actor_logits(actor_p, obs, rnn_a.reshape(-1, rnn_a.shape[-1]),
                                 avail.reshape(-1, avail.shape[-1]))
        _, old_lp, _ = categorical_stats(logits, actions.reshape(-1))

    a_tr = [actor_p[k].requires_grad_(True) for k in ACTOR_TRAINABLE]
    c_tr = [critic_p[k].requires_grad_(True) for k in CRITIC_TRAINABLE]
    opt_a = opt_a or AdamState(a_tr, args.lr, args.optim_eps)
    opt_c = opt_c or AdamState(c_tr, args.critic_lr, args.optim_eps)

    flat = dict(obs=obs, rnn_a=rnn_a.reshape(Bf * T, -1), rnn_c=rnn_c_all[:, :T].reshape(Bf * T, -1),
                act=actions.reshape(-1), avail=avail.reshape(Bf * T, -1),
                ret=returns.reshape(-1), alive=alive.reshape(-1), old_lp=old_lp,
                adv=adv.reshape(-1), old_v=cur_v.reshape(-1))
    stats = []
    for ep in range(args.ppo_epoch):
        # generate_data (:368-424): one minibatch = a permutation of the first
        # batch_size*T rows; available_actions loses its LAST EPISODE (:394) which is
        # consistent with indices < batch_size*T when batch_size <= Bf - 1.
        idx = perms[ep] if perms is not None else torch.randperm(rows)
        e = ppo_epoch(actor_p, critic_p, flat, args, idx)
        with torch.no_grad():
            n_a = opt_a.clip_step([e["grads_actor"][k] for k in ACTOR_TRAINABLE], args.max_grad_norm)
            n_c = opt_c.clip_step([e["grads_critic"][k] for k in CRITIC_TRAINABLE], args.max_grad_norm)
        stats.append(dict(value_loss=e["value_loss"].item(), policy_loss=e["policy_loss"].item(),
                          dist_entropy=e["dist_entropy"].item(), actor_grad_norm=n_a.item(),
                          critic_grad_norm=n_c.item(), ratio=e["ratio"].item(),
                          grads_actor=e["grads_actor"] if ep == 0 else None,
                          grads_critic=e["grads_critic"] if ep == 0 else None))
    for t in a_tr + c_tr:
        t.requires_grad_(False)
    pre = dict(values_all=v_all, returns=returns, advantages=adv, old_logp=old_lp.view(Bf, T))
    return stats, pre, opt_a, opt_c


# ----------------------------------------------------------------------------------
# f2  Prediction_policy.learn  (nova/prediction_policy.py:120-253), the "next" row of SURVEY §8f rank 2
# ----------------------------------------------------------------------------------
DECODER_KEYS = ["decoder.linear.weight", "decoder.linear.bias", "decoder.rnn.weight_ih_l0", "decoder.rnn.weight_hh_l0",
                "decoder.rnn.bias_ih_l0", "decoder.rnn.bias_hh_l0", "decoder.out.weight", "decoder.out.bias"]


def prediction_batch(history, attention, behavior, flag, select_idx, pred_length):
    """prediction_batch_wrapper (nova/prediction_policy.py:123-164) for one agent-net, with the sampled
    flat indices given: idx -> (episode idx // avail_len, time idx % avail_len), avail_len = T - pred_length - 1.
    history [B,T,N,o], attention [B,T,N,D], behavior [B,T,N,L], flag [B,T] (the batch's ``terminated`` column, which
    the reference multiplies the error with, :196 / :163).  Returns x0 [P,N,o], att0 [P,N,D], lat0 [P,N,L],
    target [P,N,pred_length,o], mask [P,N,pred_length,o]."""
    B, T = history.shape[:2]
    avail_len = T - pred_length - 1
    b = torch.div(select_idx, avail_len, rounding_mode="floor")
    t = select_idx % avail_len
    x0, att0, lat0 = history[b, t], attention[b, t], behavior[b, t]
    target = torch.stack([history[b, t + 1 + k] for k in range(pred_length)], dim=2)          # [P,N,pl,o]
    mask = flag[b, t].to(history.dtype).view(-1, 1, 1, 1).expand_as(target)
    return x0, att0, lat0, target, mask


def prediction_decoder(dp, last_state, hidden, pred_length, keep, p_drop):
    """Prediction_Decoder.forward with teacher_forcing_ratio = 0 (nova/prediction_net.py:37-63) around
    DecoderRNN.forward (:19-27): ReLU(linear) -> 1-step GRU -> tanh -> dropout -> out, fed back on itself.
    last_state [P,N,o]; hidden [P*N,D]; keep [pred_length, P*N, D] booleans (the dropout draw)."""
    P, N, o = last_state.shape
    h = hidden
    x = last_state.reshape(P * N, o)
    outs = []
    for t in range(pred_length):
        u = F.relu(x @ dp["decoder.linear.weight"].t() + dp["decoder.linear.bias"])
        gi = u @ dp["decoder.rnn.weight_ih_l0"].t() + dp["decoder.rnn.bias_ih_l0"]
        h = gru_cell(gi, h, dp["decoder.rnn.weight_hh_l0"], dp["decoder.rnn.bias_hh_l0"])
        y = torch.tanh(h) * keep[t].to(h.dtype) / (1.0 - p_drop)
        x = y @ dp["decoder.out.weight"].t() + dp["decoder.out.bias"]
        outs.append(x)
    return torch.stack(outs, dim=1).view(P, N, pred_length, o)


def prediction_learn_agent(gat_p, dec_p, history, attention, behavior, flag, select_idx, gumbel, keep, args, opt=None):
    """One agent-net's share of Prediction_policy.learn (:183-244): GAT forward on the sampled transitions,
    pred_length-step decoder roll-out, masked L1 loss (:228-230), separate clip_grad_norm_ of the GAT and the decoder
    gradients (:236-243), ONE Adam over both parameter lists (:84-90).  Updates the dicts in place."""
    pl, o = args.pred_length, history.shape[-1]
    x0, att0, lat0, target, mask = prediction_batch(history, attention, behavior, flag, select_idx, pl)
    P, N = x0.shape[:2]
    gat_keys = list(gat_p.keys())
    g_tr = [gat_p[k].requires_grad_(True) for k in gat_keys]
    d_tr = [dec_p[k].requires_grad_(True) for k in DECODER_KEYS]
    hidden = gat_forward(gat_p, torch.cat([x0, lat0], dim=-1), att0.reshape(P * N, -1), gumbel)
    pred = prediction_decoder(dec_p, x0, hidden, pl, keep.reshape(pl, P * N, -1), args.decoder_dropout)
    loss = ((target - pred).abs() * mask).sum() / (mask.sum() + 1e-10) * o * pl
    grads = torch.autograd.grad(loss, g_tr + d_tr)
    g_g, n_g = clip_grads(list(grads[:len(g_tr)]), args.max_grad_norm)
    g_d, n_d = clip_grads(list(grads[len(g_tr):]), args.max_grad_norm)
    opt = opt or AdamState(g_tr + d_tr, args.lr_predict, args.optim_eps)
    with torch.no_grad():
        opt.step(g_g + g_d)
    for t in g_tr + d_tr:
        t.requires_grad_(False)
    return dict(loss=float(loss.detach()), gat_grad_norm=float(n_g), dec_grad_norm=float(n_d),
                grads=dict(zip(gat_keys + DECODER_KEYS, [g.detach() for g in grads])),
                clipped=dict(zip(gat_keys + DECODER_KEYS, [g.detach() for g in g_g + g_d]))), opt


# ----------------------------------------------------------------------------------
# f3  Behavior_policy.learn  (nova/stable_behavior_policy.py:124-279), SURVEY §8f rank 3
# ----------------------------------------------------------------------------------
BEH_ENCODER_KEYS = ["linear.weight", "linear.bias", "rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0",
                    "rnn.bias_hh_l0", "out.weight", "out.bias"]


def behavior_windows(history, step, W):
    """behavior_traj_wrapper (:127-157): the W-step window ending at ``step`` (zero padded in front) and the W steps
    that follow it.  history [B,T,N,o] -> curr, next [B,N,W,o]."""
    B, T, N, o = history.shape
    start = max(0, step - W + 1)
    plug = max(0, W - step - 1)
    curr = torch.zeros(B, N, W, o, dtype=history.dtype)
    curr[:, :, plug:] = history[:, start:step + 1].permute(0, 2, 1, 3)
    nxt = history[:, step + 1:step + W + 1].permute(0, 2, 1, 3)
    return curr, nxt


def behavior_decoder(dp, curr, latent, hidden, keep, p_drop):
    """Behavior_Latent_Decoder.forward (nova/behavior_net.py:57-72) + DecoderRNN.forward (:40-47): the window with the
    latent tiled on every step -> ReLU(linear) -> GRU over the W steps from the carried hidden -> tanh -> dropout -> out.
    curr [B,N,W,o], latent [B,N,L], hidden [B*N,Hd], keep [B*N,W,Hd] -> (pred [B,N,W,o], new hidden)."""
    B, N, W, o = curr.shape
    x = torch.cat([curr, latent.unsqueeze(2).expand(B, N, W, latent.shape[-1])], dim=-1).reshape(B * N, W, -1)
    u = F.relu(x @ dp["decoder.linear.weight"].t() + dp["decoder.linear.bias"])
    h, outs = hidden, []
    for t in range(W):
        gi = u[:, t] @ dp["decoder.rnn.weight_ih_l0"].t() + dp["decoder.rnn.bias_ih_l0"]
        h = gru_cell(gi, h, dp["decoder.rnn.weight_hh_l0"], dp["decoder.rnn.bias_hh_l0"])
        outs.append(h)
    y = torch.tanh(torch.stack(outs, dim=1)) * keep.to(u.dtype) / (1.0 - p_drop)
    pred = y @ dp["decoder.out.weight"].t() + dp["decoder.out.bias"]
    return pred.view(B, N, W, o), h


def behavior_learn_agent(enc_p, dec_p, history, mask, keep, args, opt=None):
    """One agent-net's share of Behavior_policy.learn (:183-262).  history [B,T,N,o] (the batch without its last
    step), mask [B,T] (``terminated`` on Highway, ``1 - terminated`` on MPE, :186-189), keep [T-1-W, B*N, W, Hd].
    The encoder / decoder hidden states and the soft-updated latent are carried — with their graph — across all
    window positions, so the backward is one BPTT over (T-1-W) x W steps.  Updates the dicts in place."""
    B, T, N, o = history.shape
    W, L = args.max_history_len, args.latent_dim
    e_tr = [enc_p[k].requires_grad_(True) for k in BEH_ENCODER_KEYS]
    d_tr = [dec_p[k].requires_grad_(True) for k in DECODER_KEYS]
    latent = torch.zeros(B, N, L, dtype=history.dtype)
    eh = torch.zeros(B * N, args.encoder_rnn_dim, dtype=history.dtype)
    dh = torch.zeros(B * N, args.decoder_rnn_dim, dtype=history.dtype)
    n_pos = T - 1 - W
    b_err, s_err = 0.0, 0.0
    for j in range(n_pos):
        curr, nxt = behavior_windows(history, j, W)
        m_next = mask[:, j + 1:j + 1 + W].to(history.dtype).view(B, 1, W, 1).expand(B, N, W, o)
        pred, dh = behavior_decoder(dec_p, curr, latent, dh, keep[j], args.decoder_dropout)
        eh, new_latent = behavior_encoder(enc_p, curr.reshape(B * N, W, o), eh)
        stab = torch.linalg.norm(curr - pred, dim=-1).reshape(-1)
        latent = (1 - args.soft_update_coef) * latent + new_latent.view(B, N, L) * args.soft_update_coef
        err = (nxt - pred).abs() * m_next
        b_err = b_err + err.sum() / (m_next.sum() + 1e-10) * o * N
        s_err = s_err + torch.clamp(stab - args.thres_small_variation, min=0).sum() / B / W
    b_err, s_err = b_err / n_pos, s_err / n_pos
    loss = b_err + args.behavior_variation_penalty * s_err
    grads = torch.autograd.grad(loss, e_tr + d_tr)
    g_e, n_e = clip_grads(list(grads[:len(e_tr)]), args.max_grad_norm)
    g_d, n_d = clip_grads(list(grads[len(e_tr):]), args.max_grad_norm)
    opt = opt or AdamState(e_tr + d_tr, args.lr_behavior, args.optim_eps)
    with torch.no_grad():
        opt.step(g_e + g_d)
    for t in e_tr + d_tr:
        t.requires_grad_(False)
    return dict(behavior_loss=float(b_err.detach()), stability_loss=float(s_err.detach()), loss=float(loss.detach()),
                enc_grad_norm=float(n_e), dec_grad_norm=float(n_d),
                clipped=dict(zip(["enc:" + k for k in BEH_ENCODER_KEYS] + ["dec:" + k for k in DECODER_KEYS],
                                 [g.detach() for g in g_e + g_d]))), opt


# ----------------------------------------------------------------------------------
# f4  observation-history wrapper  (observation_wrapper.py:68-141), SURVEY §8f rank 4
# ----------------------------------------------------------------------------------
class ObsHistory:
    """observersation_state_history_wrapper restated without the per-slot deques: ``ids[k][i]`` is the first-seen-order
    id list (:82-88), ``win`` [B,A,N,W,o] the last W rows of every slot (:101-119), ``single`` the newest row (:124-141).
    A slot that does not exist yet has an all-zero window, so appending a zero row to it is a no-op and the update is
    one shift-and-append over all N slots."""

    def __init__(self, B, A, N, W, o):
        import numpy as np
        self.ids = [[[] for _ in range(A)] for _ in range(B)]
        self.win = np.zeros((B, A, N, W, o), dtype=np.float32)
        self.single = np.zeros((B, A, N, o), dtype=np.float32)

    def step(self, obs):
        import numpy as np
        B, A, M, od = obs.shape
        new = np.zeros_like(self.single)
        for k in range(B):
            for i in range(A):
                ids = self.ids[k][i]
                for j in range(M):
                    if np.any(obs[k, i, j, :]):                       # :80
                        vid = int(obs[k, i, j, 0])                    # :81
                        if vid not in ids:
                            ids.append(vid)                           # :84
                        new[k, i, ids.index(vid)] = obs[k, i, j, 1:]  # :90
        self.win = np.concatenate([self.win[:, :, :, 1:], new[:, :, :, None]], axis=3)
        self.single = new
        return self.win, self.single


# ----------------------------------------------------------------------------------
# f2'  GAT_Net backward written out by hand — the arithmetic the K1 backward kernels will implement
#      (checked against autograd through gat_forward in tests/test_oracle_golden.py)
# ----------------------------------------------------------------------------------
def _gru_cell_backward(gi, h_prev, w_hh, b_hh, d_h):
    """Backward of gru_cell: returns (d_gi [.,3H], d_gh [.,3H], d_h_prev [.,H]) for upstream d_h.
    d_h_prev here is only the direct (z * d_h) path plus d_gh W_hh; weight gradients are formed by the caller."""
    hd = h_prev.shape[-1]
    gh = h_prev @ w_hh.t() + b_hh
    r = torch.sigmoid(gi[..., :hd] + gh[..., :hd])
    z = torch.sigmoid(gi[..., hd:2 * hd] + gh[..., hd:2 * hd])
    n = torch.tanh(gi[..., 2 * hd:] + r * gh[..., 2 * hd:])
    d_n = d_h * (1.0 - z)
    d_z = d_h * (h_prev - n)
    da_n = d_n * (1.0 - n * n)
    d_r = da_n * gh[..., 2 * hd:]
    da_z = d_z * z * (1.0 - z)
    da_r = d_r * r * (1.0 - r)
    d_gi = torch.cat([da_r, da_z, da_n], dim=-1)
    d_gh = torch.cat([da_r, da_z, da_n * r], dim=-1)
    d_h_prev = d_h * z + d_gh @ w_hh
    return d_gi, d_gh, d_h_prev


def gat_backward_manual(p, obs, h_prev, gumbel, d_out, tau=0.01):
    """d(loss)/d(parameters of GAT_Net) for upstream gradient ``d_out`` [B*N, D] of gat_forward's output, written
    as the explicit chain of products / scatters a kernel performs (no autograd).  Returns dict keyed like ``p``."""
    B, N, _ = obs.shape
    H = p["encoding.weight"].shape[0]
    D = p["q.weight"].shape[0]
    idx = neighbour_index(N)                                                     # [N, N-1]
    g = {k: torch.zeros_like(v) for k, v in p.items()}
    # ---- forward, keeping what the backward needs -------------------------------------------------
    pre = obs @ p["encoding.weight"].t() + p["encoding.bias"]
    enc = F.relu(pre)
    dirs = []
    for sfx, order in (("", list(range(N - 1))), ("_reverse", list(range(N - 2, -1, -1)))):
        w_ih, w_hh = p["hard_bi_GRU.weight_ih_l0" + sfx], p["hard_bi_GRU.weight_hh_l0" + sfx]
        b_ih, b_hh = p["hard_bi_GRU.bias_ih_l0" + sfx], p["hard_bi_GRU.bias_hh_l0" + sfx]
        ego = enc @ w_ih[:, :H].t() + b_ih
        nbr = enc @ w_ih[:, H:].t()
        h = torch.zeros(B, N, H)
        hs = torch.empty(B, N, N - 1, H)                                         # hidden AFTER each position
        for s in order:
            h = gru_cell(ego + nbr[:, idx[:, s], :], h, w_hh, b_hh)
            hs[:, :, s] = h
        dirs.append(dict(sfx=sfx, order=order, ego=ego, nbr=nbr, hs=hs))
    hh = torch.cat([dirs[0]["hs"], dirs[1]["hs"]], dim=-1)
    logits = hh @ p["hard_encoding.weight"].t() + p["hard_encoding.bias"]
    hard = torch.sigmoid(((logits[..., 1] - logits[..., 0]) + (gumbel[..., 1] - gumbel[..., 0])) / tau)
    e2 = enc.reshape(-1, H)
    q = (e2 @ p["q.weight"].t()).view(B, N, D)
    k = (e2 @ p["k.weight"].t()).view(B, N, D)
    v_pre = (e2 @ p["v.weight"].t() + p["v.bias"]).view(B, N, D)
    v = F.relu(v_pre)
    inv = 1.0 / float(math.sqrt(D))
    kj, vj = k[:, idx, :], v[:, idx, :]                                          # [B,N,N-1,D]
    soft = torch.softmax(torch.einsum("bid,bisd->bis", q, kj) * inv, dim=-1)
    w = soft * hard
    x = torch.einsum("bis,bisd->bid", w, vj).reshape(-1, D)
    gi_c = x @ p["rnn.weight_ih"].t() + p["rnn.bias_ih"]
    # ---- backward -----------------------------------------------------------------------------------
    d_gi, d_gh, _ = _gru_cell_backward(gi_c, h_prev, p["rnn.weight_hh"], p["rnn.bias_hh"], d_out)
    g["rnn.weight_ih"] = d_gi.t() @ x; g["rnn.bias_ih"] = d_gi.sum(0)
    g["rnn.weight_hh"] = d_gh.t() @ h_prev; g["rnn.bias_hh"] = d_gh.sum(0)
    d_x = (d_gi @ p["rnn.weight_ih"]).view(B, N, D)
    d_w = torch.einsum("bid,bisd->bis", d_x, vj)                                 # [B,N,N-1]
    d_v = torch.zeros(B, N, D)
    d_v.index_add_(1, idx.reshape(-1), (w.unsqueeze(-1) * d_x.unsqueeze(2)).reshape(B, N * (N - 1), D))
    d_soft, d_hard = d_w * hard, d_w * soft
    d_score = soft * (d_soft - (soft * d_soft).sum(-1, keepdim=True)) * inv
    d_q = torch.einsum("bis,bisd->bid", d_score, kj)
    d_k = torch.zeros(B, N, D)
    d_k.index_add_(1, idx.reshape(-1), (d_score.unsqueeze(-1) * q.unsqueeze(2)).reshape(B, N * (N - 1), D))
    d_delta = d_hard * hard * (1.0 - hard) / tau                                 # d / d(l1 - l0)
    d_logits = torch.stack([-d_delta, d_delta], dim=-1)
    g["hard_encoding.weight"] = torch.einsum("bisc,bish->ch", d_logits, hh)
    g["hard_encoding.bias"] = d_logits.sum((0, 1, 2))
    d_hh = d_logits @ p["hard_encoding.weight"]                                  # [B,N,N-1,2H]
    d_enc = torch.zeros(B, N, H)
    for di, dd in enumerate(dirs):
        sfx = dd["sfx"]
        w_ih, w_hh = p["hard_bi_GRU.weight_ih_l0" + sfx], p["hard_bi_GRU.weight_hh_l0" + sfx]
        b_hh = p["hard_bi_GRU.bias_hh_l0" + sfx]
        d_hs = d_hh[..., di * H:(di + 1) * H]
        d_ego, d_nbr = torch.zeros(B, N, 3 * H), torch.zeros(B, N, 3 * H)
        gw_hh, gb_hh = torch.zeros_like(w_hh), torch.zeros_like(b_hh)
        d_h = torch.zeros(B, N, H)
        order = dd["order"]
        for pos in range(len(order) - 1, -1, -1):                                # BPTT, last position first
            s = order[pos]
            h_before = dd["hs"][:, :, order[pos - 1]] if pos > 0 else torch.zeros(B, N, H)
            d_h = d_h + d_hs[:, :, s]
            gi = dd["ego"] + dd["nbr"][:, idx[:, s], :]
            dgi, dgh, d_h = _gru_cell_backward(gi, h_before, w_hh, b_hh, d_h)
            gw_hh += torch.einsum("bng,bnh->gh", dgh, h_before); gb_hh += dgh.sum((0, 1))
            d_ego += dgi
            d_nbr.index_add_(1, idx[:, s], dgi)                                  # the neighbour part scatters to node j(i, s)
        g["hard_bi_GRU.weight_hh_l0" + sfx], g["hard_bi_GRU.bias_hh_l0" + sfx] = gw_hh, gb_hh
        g["hard_bi_GRU.weight_ih_l0" + sfx] = torch.cat([torch.einsum("bng,bnh->gh", d_ego, enc),
                                                          torch.einsum("bng,bnh->gh", d_nbr, enc)], dim=1)
        g["hard_bi_GRU.bias_ih_l0" + sfx] = d_ego.sum((0, 1))
        d_enc += d_ego @ w_ih[:, :H] + d_nbr @ w_ih[:, H:]
    d_vpre = d_v * (v_pre > 0).to(d_v.dtype)
    g["q.weight"] = d_q.reshape(-1, D).t() @ e2
    g["k.weight"] = d_k.reshape(-1, D).t() @ e2
    g["v.weight"] = d_vpre.reshape(-1, D).t() @ e2; g["v.bias"] = d_vpre.sum((0, 1))
    d_enc += d_q @ p["q.weight"] + d_k @ p["k.weight"] + d_vpre @ p["v.weight"]
    d_pre = d_enc * (pre > 0).to(d_enc.dtype)
    g["encoding.weight"] = torch.einsum("bnh,bni->hi", d_pre, obs); g["encoding.bias"] = d_pre.sum((0, 1))
    return g
