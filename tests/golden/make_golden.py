#!/usr/bin/env python
"""Generate the golden fixtures in tests/golden/ by RUNNING THE REFERENCE ITSELF.

Runs only in the build container (needs /root/reference, read-only).  It imports the
reference's own hot-path modules — nova.GAT_Net, nova.prediction_policy,
nova.stable_behavior_policy, controllers.dcntrl_controller, learners.ippo_learner,
components.episode_buffer — on the CPU, feeds them seeded synthetic inputs and
saves inputs, weights, explicit noise and outputs.  The fixtures pin the oracle
(oracle/iplan_oracle.py) and, through it and directly, the CUDA path.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py

Nothing on the GPU box reads /root/reference; only the committed *.pt files travel.
"""
import copy
import json
import os
import sys
import warnings

import numpy as np
import torch
import yaml

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(1, REPO)
warnings.filterwarnings("ignore")

from iplan_b200.config import make_args, merged_config  # noqa: E402
from obs_episode import f32_digest, obs_episode_inputs  # noqa: E402


# ---------------------------------------------------------------------------------
# config: re-derive the merged YAML config from the reference files (main.py:59-100)
# ---------------------------------------------------------------------------------
def reference_config(env):
    def load(*p):
        with open(os.path.join(REF, "config", *p)) as f:
            return yaml.safe_load(f)
    cfg = load("default.yaml")
    cfg["env"] = env                      # the key the user edits to choose the env file
    env_cfg = load("envs", "highway.yaml" if env == "highway" else "simple_spread_Hetero.yaml")
    alg_cfg = load("algs", "ippo.yaml")
    for u in (env_cfg, alg_cfg):          # recursive_dict_update: existing keys win
        for k, v in u.items():
            if k not in cfg:
                cfg[k] = v
    return cfg


class NullLogger:
    def __init__(self):
        self.stats = {}

    def log_stat(self, key, value, t):
        self.stats[key] = float(value)


def sd_clone(module):
    return {k: v.detach().clone() for k, v in module.state_dict().items()}


def ref_args(env, **over):
    a = make_args(env, use_cuda=False, device="cpu", **over)
    return a


def make_scheme(args):
    """run_ippo.py:160-180."""
    import torch as th
    from components.transforms import OneHot
    scheme = {
        "state": {"vshape": args.state_shape},
        "obs": {"vshape": args.obs_shape, "group": "agents"},
        "actions": {"vshape": (1,), "group": "agents", "dtype": th.long},
        "rnn_states_actors": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "rnn_states_critics": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "history": {"vshape": (args.max_vehicle_num, args.obs_shape_single,), "group": "agents"},
        "behavior_latent": {"vshape": (args.max_vehicle_num, args.latent_dim,), "group": "agents"},
        "attention_latent": {"vshape": (args.max_vehicle_num, args.attention_dim,), "group": "agents"},
        "avail_actions": {"vshape": (args.n_actions,), "group": "agents", "dtype": th.int},
        "reward": {"vshape": (1,), "group": "agents"},
        "speed": {"vshape": (1,), "group": "agents"},
        "terminated": {"vshape": (1,), "group": "agents", "dtype": th.uint8},
    }
    groups = {"agents": args.n_agents}
    preprocess = {"actions": ("actions_onehot", [OneHot(out_dim=args.n_actions)])}
    return scheme, groups, preprocess


def synth_history(rng, B, A, N, o, fill):
    """Highway-shaped observation rows (SURVEY §8d): col 0 presence, rest U(-1,1);
    only the first ``fill`` slots are non-zero."""
    h = rng.uniform(-1, 1, size=(B, A, N, o)).astype(np.float32)
    h[..., 0] = 1.0
    h[:, :, fill:, :] = 0.0
    return h


# ---------------------------------------------------------------------------------
def golden_config():
    out = {}
    for env in ("highway", "MPE"):
        ref = reference_config(env)
        mine = merged_config(env)
        for k, v in ref.items():
            assert k in mine and mine[k] == v, (env, k, v, mine.get(k))
        out[env] = ref
    torch.save(out, os.path.join(HERE, "config.pt"))
    print("config ok")


def golden_gat():
    from nova.GAT_Net import GAT_Net
    cases = {}
    for name, env, B, fill in (("mpe", "MPE", 3, 6), ("highway", "highway", 2, 21)):
        args = ref_args(env)
        N, o, L, D = args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim
        torch.manual_seed(1234 + B)
        net = GAT_Net(input_shape=o + L, args=args)
        rng = np.random.default_rng(7 + B)
        hist = synth_history(rng, B, 1, N, o, fill)[:, 0]
        lat = rng.dirichlet(np.ones(L), size=(B, N)).astype(np.float32)
        x = torch.tensor(np.concatenate([hist, lat], axis=-1))
        h_prev = torch.tensor(rng.uniform(-1, 1, size=(B * N, D)).astype(np.float32))
        seed = 4242
        torch.manual_seed(seed)
        with torch.no_grad():
            out = net(x, h_prev)
        torch.manual_seed(seed)
        e = torch.empty(B * N * (N - 1), 2).exponential_()
        cases[name] = dict(params=sd_clone(net), obs=x, h_prev=h_prev,
                           gumbel=(-e.log()).view(B, N, N - 1, 2), out=out.clone(),
                           dims=dict(B=B, N=N, o=o, L=L, D=D))
        print("gat", name, tuple(out.shape), float(out.abs().mean()))
    torch.save(cases, os.path.join(HERE, "gat_net.pt"))


def golden_rollout_modules():
    """Prediction_policy.GAT_latent_update, Behavior_policy.latent_update and
    DcntrlMAC.select_actions_ippo on the MPE-easy shape (BASELINE config 1) and a
    cut-down Highway shape, two consecutive steps each."""
    from nova.prediction_policy import Prediction_policy
    from nova.stable_behavior_policy import Behavior_policy
    from controllers.dcntrl_controller import DcntrlMAC
    from components.episode_buffer import EpisodeBatch

    cases = {}
    for name, env, B, over in (("mpe", "MPE", 4, {}),
                               ("highway", "highway", 2, dict(n_agents=2, n_other_vehicles=53))):
        args = ref_args(env, batch_size_run=B, **over)
        A, N, o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
        L, D, E, R, W = args.latent_dim, args.attention_dim, args.encoder_rnn_dim, args.rnn_hidden_dim, args.max_history_len
        T = 3
        args.episode_limit = T
        torch.manual_seed(99)
        logger = NullLogger()
        pred = Prediction_policy(args, logger)
        beh = Behavior_policy(args, logger)
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        mac = DcntrlMAC(batch.scheme, groups, args)
        # make the policy head non-degenerate (gain 0.01 init gives ~uniform logits)
        for ag in mac.agents:
            with torch.no_grad():
                ag.act.action_out.linear.weight.mul_(40.0)
                ag.act.action_out.linear.bias.uniform_(-0.5, 0.5)
                ag.base.feature_norm.weight.uniform_(0.5, 1.5)
                ag.base.feature_norm.bias.uniform_(-0.2, 0.2)
        for cr in mac.critics:
            with torch.no_grad():
                cr.base.feature_norm.weight.uniform_(0.5, 1.5)
                cr.base.feature_norm.bias.uniform_(-0.2, 0.2)

        rng = np.random.default_rng(2024)
        fills = [min(N, 4 + 2 * t) if env == "highway" else N for t in range(W + 2)]
        singles = [synth_history(rng, B, A, N, o, fills[t]).astype(np.float64) for t in range(W + 2)]

        def window(t):
            w = np.zeros((B, A, N, W, o), dtype=np.float64)
            for k in range(W):
                src = t - (W - 1 - k)
                if src >= 0:
                    w[:, :, :, k] = singles[src]
            return w

        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   gat=[sd_clone(m) for m in pred.pred_GAT],
                   beh=[sd_clone(m) for m in beh.behavior_encoder],
                   actors=[sd_clone(m) for m in mac.agents],
                   critics=[sd_clone(m) for m in mac.critics], steps=[])

        rnn_a = np.zeros((B, 1, A, R), dtype=np.float32)
        rnn_c = np.zeros_like(rnn_a)
        enc_rnn = np.zeros((B, 1, A, N, E), dtype=np.float32)
        beh_lat = np.zeros((B, A, N, L), dtype=np.float32)
        att = np.zeros((B, A, N, D), dtype=np.float32)
        avail = np.ones((B, A, args.n_actions), dtype=np.int64)
        avail[0, 0, 1] = 0                                   # exercise the -1e10 mask

        for t in range(3):
            step = dict(history_single=singles[t].copy(), window=window(t).copy(),
                        att_in=np.array(att), beh_in=np.array(beh_lat),
                        enc_rnn_in=np.array(enc_rnn))
            seed = 555 + t
            torch.manual_seed(seed)
            att = pred.GAT_latent_update(singles[t], att, beh_lat)
            torch.manual_seed(seed)
            rows = B * N * (N - 1)
            step["gumbel"] = torch.stack(
                [(-torch.empty(rows, 2).exponential_().log()).view(B, N, N - 1, 2) for _ in range(A)])
            step["att_out"] = np.array(att)
            if t > 0:
                # the runner updates the behaviour latent after the GAT (runner :222-231)
                beh_lat, enc_rnn_t = beh.latent_update(window(t), enc_rnn, beh_lat)
                enc_rnn = enc_rnn_t.detach().numpy()
                step["beh_out"] = np.array(beh_lat)
                step["enc_rnn_out"] = np.array(enc_rnn)
            pre = {"avail_actions": avail, "rnn_states_actors": rnn_a, "rnn_states_critics": rnn_c,
                   "history": singles[t], "behavior_latent": beh_lat, "attention_latent": att}
            batch.update(pre, ts=t)
            step["inputs"] = mac._build_inputs(batch, t).clone()
            step["rnn_a_in"] = rnn_a.copy()
            step["rnn_c_in"] = rnn_c.copy()
            with torch.no_grad():
                values, actions, logps, rnn_a, rnn_c = mac.select_actions_ippo(batch, t_ep=t, test_mode=True)
            step.update(values=values.copy(), actions=actions.copy(),
                        logp=torch.cat(logps, dim=1).squeeze(1).detach().clone()
                        if logps[0].dim() == 3 else torch.cat(logps, dim=-1).detach().clone(),
                        rnn_a_out=rnn_a.copy(), rnn_c_out=rnn_c.copy())
            batch.update({"actions": actions}, ts=t, mark_filled=False)
            rec["steps"].append(step)
        rec["avail"] = avail
        cases[name] = rec
        print("rollout", name, "F =", step["inputs"].shape[-1], "values", step["values"].ravel()[:3])
    torch.save(cases, os.path.join(HERE, "rollout_modules.pt"))


def golden_learner():
    """IPPOLearner.insert_episode_batch + train on seeded EpisodeBatch contents.
    Case "mpe": BASELINE config 1 dims (A=3, N=6, F=272), T=6, Bf=4, batch_size=3,
    15 epochs.  Case "highway": N=55 slots, one agent (F=2481), T=4, Bf=3, 4 epochs."""
    from controllers.dcntrl_controller import DcntrlMAC
    from learners.ippo_learner import IPPOLearner
    from components.episode_buffer import EpisodeBatch

    cases = {}
    for name, env, over in (
            ("mpe", "MPE", dict(episode_length=6, buffer_size=4, batch_size=3, batch_size_run=4)),
            ("highway", "highway", dict(n_agents=1, n_other_vehicles=54, episode_limit=4,
                                        buffer_size=3, batch_size=2, batch_size_run=3, ppo_epoch=4))):
        args = ref_args(env, **over)
        A, N, o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
        L, D, R, T, B = args.latent_dim, args.attention_dim, args.rnn_hidden_dim, args.episode_limit, args.batch_size_run
        torch.manual_seed(31337)
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        mac = DcntrlMAC(batch.scheme, groups, args)
        logger = NullLogger()
        learner = IPPOLearner(mac, batch.scheme, logger, args)
        with torch.no_grad():
            for ag in mac.agents:
                ag.act.action_out.linear.weight.mul_(30.0)
                ag.base.feature_norm.weight.uniform_(0.5, 1.5)
                ag.base.feature_norm.bias.uniform_(-0.2, 0.2)
            for cr in mac.critics:
                cr.base.feature_norm.weight.uniform_(0.5, 1.5)
                cr.base.feature_norm.bias.uniform_(-0.2, 0.2)

        rng = np.random.default_rng(77)
        data = dict(
            history=np.stack([synth_history(rng, B, A, N, o, min(N, 3 + 2 * t)) for t in range(T + 1)], axis=1),
            attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
            behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
            rnn_states_actors=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
            rnn_states_critics=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
            actions=rng.integers(0, args.n_actions, size=(B, T + 1, A, 1)),
            avail_actions=np.ones((B, T + 1, A, args.n_actions), dtype=np.int64),
            reward=rng.normal(size=(B, T + 1, A, 1)).astype(np.float32) * 3.0,
        )
        data["avail_actions"][0, 1, 0, (data["actions"][0, 1, 0, 0] + 1) % args.n_actions] = 0
        term = np.zeros((B, T + 1, A, 1), dtype=np.uint8)
        term[1, T - 2:, 0] = 1                               # agent 0 of env 1 dies near the end
        if A > 1:
            term[0, 2:, 1] = 1
        data["terminated"] = term
        batch.update(data, bs=slice(None), ts=slice(None))
        learner.insert_episode_batch(batch)

        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   data={k: torch.as_tensor(v) for k, v in data.items()},
                   actors_before=[sd_clone(m) for m in mac.agents],
                   critics_before=[sd_clone(m) for m in mac.critics])

        # pre-update quantities, per agent, through the reference's own methods
        pre = []
        for a in range(A):
            b = learner.buffers[a].get_batch()
            obs_all = mac._build_inputs_ippo(a, b, b["actions_onehot"])
            with torch.no_grad():
                ret = learner.compute_returns(a, obs_all, b["reward"][:, :-1], b["terminated_masks"],
                                              b["rnn_states_critic"]).clone()
                cur = mac.get_value_ippo(a, obs_all[:, :-1], b["rnn_states_critic"][:, :-1]).clone()
                v_all = mac.get_value_ippo(a, obs_all, b["rnn_states_critic"]).clone()
                adv = ret - cur
                adv[b["terminated_masks"][:, :-1] == 0.0] = 0.0
                std, mean = torch.std_mean(adv)
                adv = (adv - mean) / (std + 1e-5)
                lp, ent = mac.eval_action_ippo(a, obs_all[:, :-1], b["actions"][:, :-1],
                                               b["available_actions"][:, :-1], b["rnn_states_actor"][:, :-1])
            pre.append(dict(obs_all=obs_all.clone(), returns=ret.squeeze(-1), values_all=v_all.squeeze(-1),
                            advantages=adv.squeeze(-1), old_logp=lp.squeeze(-1).clone(), entropy=float(ent)))
        rec["pre"] = pre

        seed = 2718
        torch.manual_seed(seed)
        learner.train(t_env=0)
        torch.manual_seed(seed)
        rows = args.batch_size * T
        rec["perms"] = [[torch.randperm(rows) for _ in range(args.ppo_epoch)] for _ in range(A)]
        rec["actors_after"] = [sd_clone(m) for m in mac.agents]
        rec["critics_after"] = [sd_clone(m) for m in mac.critics]
        rec["stats"] = dict(logger.stats)
        rec["actor_opt_steps"] = [int(len(o.state_dict()["state"])) for o in learner.actor_optimizers]
        cases[name] = rec
        print("learner", name, {k.split("_H_")[-1]: round(v, 6) for k, v in logger.stats.items()})
    torch.save(cases, os.path.join(HERE, "learner.pt"))


def golden_prediction_learn():
    """Prediction_policy.learn (nova/prediction_policy.py:168-253) — one call on a seeded EpisodeBatch.
    The random draws of the call are recorded while the reference runs: the sampled (episode, time) indices
    (np.random.choice, :147), the Gumbel noise of GAT_Net.forward (F.gumbel_softmax, GAT_Net.py:93 — wrapped by a
    recorder that does the same arithmetic as torch's implementation) and the decoder's dropout masks
    (nn.Dropout in train mode, prediction_net.py:18,27 — read off a forward hook).
    Case "mpe": A=3, N=6, 4 episodes x T=12, pred_batch 8.  Case "highway": one agent, N=55, 3 episodes x T=12, pred_batch 6."""
    import torch.nn.functional as Fn
    from nova.prediction_policy import Prediction_policy
    from components.episode_buffer import EpisodeBatch

    cases = {}
    for name, env, over in (
            ("mpe", "MPE", dict(episode_length=12, batch_size_run=4, pred_batch_size=8)),
            ("highway", "highway", dict(n_agents=1, n_other_vehicles=54, episode_limit=12, batch_size_run=3, pred_batch_size=6))):
        args = ref_args(env, **over)
        A, N, o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
        L, D, T, B = args.latent_dim, args.attention_dim, args.episode_limit, args.batch_size_run
        torch.manual_seed(99 + N)
        logger = NullLogger()
        pol = Prediction_policy(args, logger)
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        rng = np.random.default_rng(2024 + N)
        data = dict(
            history=np.stack([synth_history(rng, B, A, N, o, min(N, 3 + 2 * t)) for t in range(T + 1)], axis=1),
            attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
            behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
        )
        term = np.ones((B, T + 1, A, 1), dtype=np.uint8)       # the reference multiplies the error by this flag (:196, :163)
        term[0, 3:6, 0] = 0
        term[B - 1, :2, A - 1] = 0
        data["terminated"] = term
        batch.update(data, bs=slice(None), ts=slice(None))

        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   data={k: torch.as_tensor(v) for k, v in data.items()},
                   gat_before=[sd_clone(m) for m in pol.pred_GAT], dec_before=[sd_clone(m) for m in pol.pred_decoder])

        gumbels, drop_masks = [], [[] for _ in range(A)]
        orig_gs = Fn.gumbel_softmax

        def recording_gumbel_softmax(logits, tau=1, hard=False, eps=1e-10, dim=-1):
            assert not hard
            g = -torch.empty_like(logits).exponential_().log()       # torch/nn/functional.py gumbel_softmax
            gumbels.append(g.detach().clone())
            return ((logits + g) / tau).softmax(dim)

        hooks = []
        for i in range(A):
            def hook(mod, inp, out, i=i):
                x = inp[0].detach()
                assert bool((x != 0).all())
                drop_masks[i].append((out.detach() != 0).clone())
            hooks.append(pol.pred_decoder[i].decoder.dropout.register_forward_hook(hook))

        seed = 1618
        np.random.seed(seed)
        torch.manual_seed(seed)
        Fn.gumbel_softmax = recording_gumbel_softmax
        try:
            losses = pol.learn(batch, t_env=0)
        finally:
            Fn.gumbel_softmax = orig_gs
            for h in hooks:
                h.remove()
        # replay the numpy stream: per agent one choice(...) then pred_length x random() (prediction_net.py:55)
        np.random.seed(seed)
        avail_len = T - args.pred_length - 1
        idx = []
        for i in range(A):
            idx.append(torch.as_tensor(np.random.choice(B * avail_len, size=args.pred_batch_size, replace=False)))
            for _ in range(args.pred_length):
                np.random.random()
        assert len(gumbels) == A and all(len(m) == args.pred_length for m in drop_masks)
        rec.update(select_idx=idx, gumbel=[g.view(args.pred_batch_size, N, N - 1, 2) for g in gumbels],
                   dropout_keep=[torch.stack(m) for m in drop_masks],
                   losses=[float(x) for x in losses], stats=dict(logger.stats),
                   gat_after=[sd_clone(m) for m in pol.pred_GAT], dec_after=[sd_clone(m) for m in pol.pred_decoder],
                   # .grad after learn() = the gradients as clipped in place by clip_grad_norm_ (:236-243)
                   gat_grads=[{k: v.grad.detach().clone() for k, v in m.named_parameters()} for m in pol.pred_GAT],
                   dec_grads=[{k: v.grad.detach().clone() for k, v in m.named_parameters()} for m in pol.pred_decoder])
        cases[name] = rec
        print("prediction.learn", name, [round(float(x), 6) for x in losses])
    torch.save(cases, os.path.join(HERE, "prediction_learn.pt"))


def golden_behavior_learn():
    """Behavior_policy.learn (nova/stable_behavior_policy.py:161-279) — one call on a seeded EpisodeBatch.  The only
    random draw is the decoder's dropout (behavior_net.py:37,46; train mode), read off a forward hook.
    Case "mpe": A=3, N=6, 3 episodes x T=15 (4 window positions).  Case "highway": one agent, N=55, 2 episodes x T=13."""
    from nova.stable_behavior_policy import Behavior_policy
    from components.episode_buffer import EpisodeBatch

    cases = {}
    for name, env, over in (
            ("mpe", "MPE", dict(episode_length=15, batch_size_run=3)),
            ("highway", "highway", dict(n_agents=1, n_other_vehicles=54, episode_limit=13, batch_size_run=2))):
        args = ref_args(env, **over)
        A, N, o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
        L, D, T, B = args.latent_dim, args.attention_dim, args.episode_limit, args.batch_size_run
        torch.manual_seed(555 + N)
        logger = NullLogger()
        pol = Behavior_policy(args, logger)
        scheme, groups, preprocess = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=preprocess, device="cpu")
        rng = np.random.default_rng(4048 + N)
        data = dict(
            history=np.stack([synth_history(rng, B, A, N, o, min(N, 3 + 2 * t)) for t in range(T + 1)], axis=1),
            behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
        )
        term = np.zeros((B, T + 1, A, 1), dtype=np.uint8)
        term[0, 11:, 0] = 1
        term[B - 1, 12:, A - 1] = 1
        if env != "MPE":
            term = 1 - term        # highway: the flag is used as the mask directly (:186-189)
        data["terminated"] = term.astype(np.uint8)
        batch.update(data, bs=slice(None), ts=slice(None))
        rec = dict(args={k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                   data={k: torch.as_tensor(v) for k, v in data.items()},
                   enc_before=[sd_clone(m) for m in pol.behavior_encoder], dec_before=[sd_clone(m) for m in pol.behavior_decoder])
        drop = [[] for _ in range(A)]
        hooks = []
        for i in range(A):
            def hook(mod, inp, out, i=i):
                assert bool((inp[0].detach() != 0).all())
                drop[i].append((out.detach() != 0).clone())
            hooks.append(pol.behavior_decoder[i].decoder.dropout.register_forward_hook(hook))
        torch.manual_seed(2236)
        try:
            b_loss, s_loss, t_loss = pol.learn(batch, t_env=0)
        finally:
            for h in hooks:
                h.remove()
        rec.update(dropout_keep=[torch.stack(m) for m in drop],
                   behavior_loss=[float(x) for x in b_loss], stability_loss=[float(x) for x in s_loss],
                   total_loss=[float(x) for x in t_loss], stats=dict(logger.stats),
                   enc_after=[sd_clone(m) for m in pol.behavior_encoder], dec_after=[sd_clone(m) for m in pol.behavior_decoder],
                   enc_grads=[{k: v.grad.detach().clone() for k, v in m.named_parameters()} for m in pol.behavior_encoder],
                   dec_grads=[{k: v.grad.detach().clone() for k, v in m.named_parameters()} for m in pol.behavior_decoder])
        cases[name] = rec
        print("behavior.learn", name, [round(float(x), 6) for x in b_loss], [round(float(x), 6) for x in s_loss])
    torch.save(cases, os.path.join(HERE, "behavior_learn.pt"))


def golden_obs_wrapper():
    """observersation_state_history_wrapper (observation_wrapper.py): 14 timesteps of synthetic raw observations in
    which vehicles enter, leave and re-enter the agents' view; records every step's obs_history_output and
    obs_single_history_output."""
    from observation_wrapper import observersation_state_history_wrapper as RefWrapper
    args = ref_args("highway", batch_size_run=3)
    B, A, N, W, o = 3, args.n_agents, args.max_vehicle_num, args.max_history_len, args.obs_shape_single
    M = 15                                                   # n_obs_vehicles (config/envs/highway.yaml:8)
    wr = RefWrapper(args, A, N, args.episode_limit, W)
    rng = np.random.default_rng(31)
    steps = []
    pool = np.arange(1000, 1000 + 40)                        # vehicle ids an agent may meet (< N distinct)
    for t in range(14):
        obs = np.zeros((B, A, M, o + 1))
        for k in range(B):
            for i in range(A):
                n_seen = rng.integers(3, M + 1)
                seen = rng.choice(pool[:20 + t], size=n_seen - 1, replace=False)
                obs[k, i, 0, 0] = 7 + i                      # ego first (:73)
                obs[k, i, 0, 1:] = rng.uniform(-1, 1, size=o)
                obs[k, i, 1:n_seen, 0] = seen
                obs[k, i, 1:n_seen, 1:] = rng.uniform(-1, 1, size=(n_seen - 1, o))
        if t == 0:
            wr.agent_obs_profile_init(obs)
        wr.obs_history_create(obs)
        single = wr.obs_single_history_output().copy()
        window = wr.obs_history_output().copy()
        steps.append(dict(obs=torch.tensor(obs, dtype=torch.float32), single=torch.tensor(single, dtype=torch.float32),
                          window=torch.tensor(window, dtype=torch.float32)))
    ids = [[list(wr.obs_vehicle_id[k][i]) for i in range(A)] for k in range(B)]
    torch.save(dict(dims=dict(B=B, A=A, N=N, W=W, o=o, M=M), steps=steps, ids=ids), os.path.join(HERE, "obs_wrapper.pt"))
    print("obs_wrapper: slots used", max(len(x) for r in ids for x in r))


def golden_obs_wrapper_episode():
    """The reference wrapper over a whole 91-observation episode (more observations than the deque's maxlen): digests of
    every timestep's obs_single_history_output / obs_history_output, of the final obs_history_episode_output(mask), and
    the slot tables.  Inputs from obs_episode_inputs(np.random.default_rng(99), ...)."""
    from observation_wrapper import observersation_state_history_wrapper as RefWrapper
    B, M = 4, 15
    args = ref_args("highway", batch_size_run=B)
    A, N, W, o, L = args.n_agents, args.max_vehicle_num, args.max_history_len, args.obs_shape_single, args.episode_limit
    wr = RefWrapper(args, A, N, L, W)
    steps, mask = obs_episode_inputs(np.random.default_rng(99), B, A, N, M, o, L)
    rec = dict(dims=dict(B=B, A=A, N=N, W=W, o=o, M=M, L=L), obs=[], single=[], window=[])
    for t, obs in enumerate(steps):
        if t == 0:
            wr.agent_obs_profile_init(obs)
        wr.obs_history_create(obs)
        rec["obs"].append(f32_digest(obs))
        rec["single"].append(f32_digest(wr.obs_single_history_output()))
        rec["window"].append(f32_digest(wr.obs_history_output()))
    rec["ids"] = [[list(map(int, wr.obs_vehicle_id[k][i])) for i in range(A)] for k in range(B)]
    raw, ep = wr.obs_history_episode_output(mask)
    rec["raw"], rec["ep"] = f32_digest(raw), f32_digest(ep)
    with open(os.path.join(HERE, "obs_wrapper_episode.json"), "w") as f:
        json.dump(rec, f, indent=0)
    print("obs_wrapper_episode:", len(steps), "steps")


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_config()
    golden_gat()
    golden_rollout_modules()
    golden_learner()
    golden_prediction_learn()
    golden_behavior_learn()
    golden_obs_wrapper()
    golden_obs_wrapper_episode()
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".pt"):
            print(f, os.path.getsize(os.path.join(HERE, f)) // 1024, "KiB")
