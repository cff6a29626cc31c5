"""IPPO learner — host-side mirror of the reference's ``IPPOLearner``
(/root/reference/learners/ippo_learner.py:17-424).  The arithmetic is csrc/learner.cu:
K2a (GAE scan + advantage moments), the fused forward, K2b (PPO losses + backward through
heads / LayerNorm / GRU gates), the fc1 products over the packed episode rows, gradient-norm
clipping and Adam.  All agents are updated in the same launches (they are independent
parameter sets; the reference loops over them, :249).

Same constructor ``IPPOLearner(mac, scheme, logger, args)`` and public methods
(``insert_episode_batch``, ``train``, ``cuda``, ``save_models``, ``load_models``,
``lr_decay``, ``compute_returns``); logs the same six statistics under the same keys.

Multi-GPU (new capability, SURVEY §8e): environments are sharded across ranks, each
rank keeps its own episodes; per ``train()`` one all-reduce of the advantage moments and
mask sums, and per PPO epoch ONE all-reduce (SUM) of the concatenated actor+critic
gradient buffer over NCCL.  Loss denominators, the advantage mean/std and the clip norm
are global quantities, so N ranks x B/N envs reproduce one rank x B envs.
"""
import copy
import math

import torch as th

from .. import _lib, parallel
from ..modules.flat import DEAD, FROZEN, POPART_KEYS


class _AdamSlot:
    """torch.optim.Adam-compatible ``state_dict`` view of one agent's slice of the flat
    optimiser state (files ``actor_{i}_opt.th`` / ``critic_{i}_opt.th``, reference :322-326).
    Only tensors that ever receive a gradient carry state (18 of the 22/26 tensors)."""

    def __init__(self, owner, kind, index):
        self.owner, self.kind, self.index = owner, kind, index

    def _entries(self, cuda_format=None):
        """(param id, name, shape, offset, numel) in torch's parameter order.  In the CUDA reference's format the
        critic has no v_out.* parameters (modules/flat.py POPART_KEYS): ids run over the 20 trunk tensors only."""
        stack = self.owner.stacks[self.kind]
        if cuda_format is None:
            cuda_format = self.owner.popart_cuda_quirk
        out, pi = [], 0
        for (name, shape), off in zip(stack.spec, stack.offsets):
            if cuda_format and self.kind == "critic" and name in POPART_KEYS:
                continue
            n = int(math.prod(shape)) if len(shape) else 1
            out.append((pi, name, shape, off, n))
            pi += 1
        return out

    def state_dict(self):
        o = self.owner
        st = {}
        for pi, name, shape, off, n in self._entries():
            if name in FROZEN or name.startswith(DEAD[0]) or o.steps[self.kind] == 0:
                continue
            if o.popart_cuda_quirk and name in POPART_KEYS:
                continue
            st[pi] = {"step": th.tensor(float(o.steps[self.kind])),
                      "exp_avg": o.exp_avg[self.kind][self.index, off:off + n].view(shape).detach().cpu().clone(),
                      "exp_avg_sq": o.exp_avg_sq[self.kind][self.index, off:off + n].view(shape).detach().cpu().clone()}
        group = {"lr": o.lrs[self.kind], "betas": (0.9, 0.999), "eps": o.optim_eps, "weight_decay": o.weight_decay,
                 "amsgrad": False, "maximize": False, "foreach": None, "capturable": False,
                 "differentiable": False, "fused": None, "params": [e[0] for e in self._entries()]}
        return {"state": st, "param_groups": [group]}

    def load_state_dict(self, sd):
        o = self.owner
        # parameter ids are positional: pick the format (26 critic params = CPU reference, 20 = CUDA reference) by count
        n_params = len(sd["param_groups"][0]["params"])
        fmt = None
        if self.kind == "critic":
            fmt = n_params == len(self._entries(cuda_format=True))
        for pi, name, shape, off, n in self._entries(cuda_format=fmt):
            if pi in sd["state"]:
                s = sd["state"][pi]
                o.exp_avg[self.kind][self.index, off:off + n] = s["exp_avg"].reshape(-1).to(o.device)
                o.exp_avg_sq[self.kind][self.index, off:off + n] = s["exp_avg_sq"].reshape(-1).to(o.device)
                o.steps[self.kind] = int(s["step"])
        o.lrs[self.kind] = sd["param_groups"][0]["lr"]


class IPPOLearner:
    def __init__(self, mac, scheme, logger, args):
        if not args.use_cuda:
            raise RuntimeError("iplan_b200.IPPOLearner runs on CUDA only (no CPU path); set args.use_cuda=True")
        self.device = th.device("cuda")
        self.args = args
        self.mac = mac
        self.logger = logger
        self.log_prefix = args.log_prefix
        self.log_stats_t = -args.learner_log_interval - 1
        self.n_agents = args.n_agents
        self.t_max = args.t_max
        self.episode_limit = args.episode_limit
        self.batch_size_run = args.batch_size_run
        self.batch_size = args.batch_size
        self.buffer_size = args.buffer_size
        self.n_actions = args.n_actions
        self.lr, self.critic_lr = args.lr, args.critic_lr
        self.use_linear_lr_decay = args.use_linear_lr_decay
        self.optim_eps, self.weight_decay = args.optim_eps, args.weight_decay
        for flag in ("use_gae", "use_clipped_value_loss", "use_huber_loss", "use_value_active_masks",
                     "use_policy_active_masks", "use_max_grad_norm", "use_recurrent_policy"):
            if not getattr(args, flag):
                raise NotImplementedError(f"only the reference's default IPPO setting is built ({flag}=True)")
        assert args.num_mini_batch == 1 and args.weight_decay == 0
        self.clip_param, self.ppo_epoch = args.clip_param, args.ppo_epoch
        self.value_loss_coef, self.entropy_coef = args.value_loss_coef, args.entropy_coef
        self.max_grad_norm, self.huber_delta = args.max_grad_norm, args.huber_delta
        self.gamma, self.gae_lambda = args.gamma, args.gae_lambda

        self.stacks = {"actor": mac.actor_stack, "critic": mac.critic_stack}
        self.exp_avg = {k: th.zeros_like(s.flat) for k, s in self.stacks.items()}
        self.exp_avg_sq = {k: th.zeros_like(s.flat) for k, s in self.stacks.items()}
        # True: behave like a CUDA run of the reference (PopArt value head never registered: frozen, absent from checkpoints)
        self.popart_cuda_quirk = bool(getattr(args, "popart_cuda_quirk", False))
        frozen = {"actor": (), "critic": ("v_out.weight", "v_out.bias") if self.popart_cuda_quirk else ()}
        self.masks = {k: s.trainable_mask(frozen[k]).to(self.device) for k, s in self.stacks.items()}
        self.steps = {"actor": 0, "critic": 0}
        self.lrs = {"actor": self.lr, "critic": self.critic_lr}
        self.actor_optimizers = [_AdamSlot(self, "actor", i) for i in range(self.n_agents)]
        self.critic_optimizers = [_AdamSlot(self, "critic", i) for i in range(self.n_agents)]
        self.actor_params = mac.parameters()
        self.critic_params = mac.critic_parameters()

        self.F = mac.input_shape
        self.T1 = self.episode_limit + 1
        self.count = 0              # episodes currently held (SeparatedReplayBuffer deque length)
        self.store = None
        self.work = None
        self.last_pre = None        # pre-update tensors of the last train() (parity tests)
        self.keep_pre = False
        self.bucket = parallel.GradBucket()
        self.grad_scale = 1.0
        self.use_dist = True        # False: ignore an active process group (single-rank reference runs in tests)

    # ------------------------------------------------------------------------------
    def lr_decay(self, episode, episodes):
        """update_linear_schedule (utils/mappo_utils/util.py:27-31)."""
        self.lrs["actor"] = self.lr - self.lr * (episode / float(episodes))
        self.lrs["critic"] = self.critic_lr - self.critic_lr * (episode / float(episodes))

    def cuda(self):
        self.mac.cuda()

    # ------------------------------------------------------------------------------
    def _alloc_store(self, Fp):
        A, Bf, T1, R, nA, dev = self.n_agents, self.buffer_size, self.T1, self.args.rnn_hidden_dim, self.n_actions, self.device
        self.store = dict(
            X=th.zeros(A, Bf, T1, Fp, device=dev), rnn_a=th.zeros(A, Bf, T1, R, device=dev),
            rnn_c=th.zeros(A, Bf, T1, R, device=dev), actions=th.zeros(A, Bf, T1, dtype=th.int32, device=dev),
            avail=th.ones(A, Bf, T1, nA, dtype=th.uint8, device=dev), reward=th.zeros(A, Bf, T1, device=dev),
            alive=th.ones(A, Bf, T1, device=dev))

    def insert_episode_batch(self, ep_batch):
        """Reference :96-126 + SeparatedReplayBuffer.insert (separated_buffer.py:47-68): append
        the batch's episodes (per-agent slices) to the buffer; ``terminated_mask = 1 - terminated``."""
        packed = getattr(ep_batch, "packed", None)
        if packed is None:
            rows = th.stack([self.mac._build_inputs_ippo(a, {k: ep_batch[k][:, :, a] for k in
                                                           ("history", "attention_latent", "behavior_latent")},
                                                         ep_batch["actions_onehot"][:, :, a])
                             for a in range(self.n_agents)]).to(self.device, th.float32)
            Fp = (self.F + 31) // 32 * 32
            X = th.zeros(*rows.shape[:-1], Fp, device=self.device)
            X[..., :self.F] = rows
        else:
            X, Fp = packed, packed.shape[-1]
        B = X.shape[1]
        if self.store is None or self.store["X"].shape[-1] != Fp:
            self._alloc_store(Fp)
        Bf = self.buffer_size
        first = max(0, B - Bf)       # deque(maxlen): of a batch longer than the buffer only the last Bf episodes survive
        nb = B - first
        over = self.count + nb - Bf
        if over > 0:                 # the oldest episodes fall out
            keep = self.count - over
            if keep > 0:
                for v in self.store.values():
                    v[:, :keep] = v[:, over:self.count].clone()
            self.count = keep
        sl = slice(self.count, self.count + nb)
        dev = self.device
        s = self.store
        s["X"][:, sl] = X[:, first:]
        s["rnn_a"][:, sl] = ep_batch["rnn_states_actors"][first:].to(dev).permute(2, 0, 1, 3)
        s["rnn_c"][:, sl] = ep_batch["rnn_states_critics"][first:].to(dev).permute(2, 0, 1, 3)
        s["actions"][:, sl] = ep_batch["actions"][first:].to(dev)[..., 0].permute(2, 0, 1).to(th.int32)
        s["avail"][:, sl] = (ep_batch["avail_actions"][first:].to(dev) != 0).permute(2, 0, 1, 3).to(th.uint8)
        s["reward"][:, sl] = ep_batch["reward"][first:].to(dev)[..., 0].permute(2, 0, 1)
        s["alive"][:, sl] = 1.0 - ep_batch["terminated"][first:].to(dev)[..., 0].permute(2, 0, 1).float()
        self.count += nb

    def can_sample(self):
        return self.count == self.buffer_size

    # ------------------------------------------------------------------------------
    def _work_buffers(self, A, rows, Fp):
        key = (A, rows, Fp)
        if self.work is None or self.work["key"] != key:
            dev = self.device
            z = lambda *s, **k: th.zeros(*s, device=dev, **k)
            hz = lambda *s: th.zeros(*s, device=dev, dtype=th.float16)
            self.work = dict(
                key=key, stat=z(A, rows, 2), Wh=hz(A, 128, Fp), Wl=hz(A, 128, Fp), ws=z(A, 128), cc=z(A, 128), Z1=z(A, rows, 128),
                Xh=hz(A, rows, Fp), Xl=hz(A, rows, Fp), Dh=hz(A, rows, 128), Dl=hz(A, rows, 128), gscale=z(2 * A),
                A1=z(A, 2, rows, 64), Z2=z(A, 2, rows, 64), A2=z(A, 2, rows, 64), GI=z(A, 2, rows, 192), GH=z(A, 2, rows, 192),
                SM=z(A, 2, 128), G=z(A, 128, Fp), logp=z(A, rows), ent=z(A, rows), value=z(A, rows),
                returns=z(A, rows), adv=z(A, rows), moments=z(A, 4, dtype=th.float64), norm=z(A, 4),
                stats=z(A, 8), sq=z(A),
                grads={k: th.zeros_like(s.flat) for k, s in self.stacks.items()})
        return self.work

    def _ctx(self, w, s, A, n_eps, T1, n_train, actor, critic, rnn_a, rnn_c, rnn_sa, rnn_ld, actions, avail, F):
        c = _lib.LearnerCtx()
        P = _lib.ptr
        c.actor, c.critic = P(actor), P(critic)
        c.actor_stride, c.critic_stride = self.stacks["actor"].stride(), self.stacks["critic"].stride()
        c.g_actor, c.g_critic = P(w["grads"]["actor"]), P(w["grads"]["critic"])
        c.feat_dim, c.n_actions, c.n_agents, c.T1, c.n_eps, c.n_train_eps = F, self.n_actions, A, T1, n_eps, n_train
        c.rnn_a, c.rnn_c, c.rnn_stride_agent, c.rnn_ld = P(rnn_a), P(rnn_c), rnn_sa, rnn_ld
        c.actions, c.avail = P(actions), P(avail)
        for k in ("Z1", "A1", "Z2", "A2", "GI", "GH", "SM"):
            setattr(c, k, P(w[k]))
        c.stat = P(w["stat"])
        c.logp_out, c.ent_out, c.value_out = P(w["logp"]), P(w["ent"]), P(w["value"])
        c.old_logp, c.old_value = P(w.get("old_logp")), P(w.get("old_value"))
        c.returns, c.adv_raw = P(w["returns"]), P(w["adv"])
        c.alive = P(s["alive"]) if s else None
        c.norm, c.stats = P(w["norm"]), P(w["stats"])
        c.clip, c.ent_coef, c.v_coef, c.huber_delta = self.clip_param, self.entropy_coef, self.value_loss_coef, self.huber_delta
        c.grad_scale = self.grad_scale
        return c

    def _mark(self, tag):
        """Optional CUDA-event timeline of the update (bench.py sets ``self.events = []``)."""
        ev = getattr(self, "events", None)
        if ev is not None:
            e = th.cuda.Event(enable_timing=True)
            e.record()
            ev.append((tag, e))

    def _forward(self, w, ctx, X, A, rows, Fp, F, actor, critic, train):
        lib, st = _lib.lib, _lib.stream()
        self._mark("fc1_fwd")
        _lib.check(lib.iplan_learner_fc1_forward(
            _lib.ptr(actor), self.stacks["actor"].stride(), _lib.ptr(critic), self.stacks["critic"].stride(),
            _lib.ptr(w["Xh"]), _lib.ptr(w["Xl"]), w["Xh"].stride(0), Fp, F, rows, A, _lib.ptr(w["stat"]),
            _lib.ptr(w["Wh"]), _lib.ptr(w["Wl"]), _lib.ptr(w["ws"]), _lib.ptr(w["cc"]), _lib.ptr(w["Z1"]), st), "fc1_forward")
        import ctypes
        self._mark("tail_train" if train else "tail_eval")
        _lib.check(lib.iplan_learner_tail(ctypes.byref(ctx), 1 if train else 0, st), "learner_tail")
        self._mark("end")

    # ------------------------------------------------------------------------------
    def train(self, t_env):
        """Reference :227-317.  Silently returns unless the buffer holds exactly
        ``buffer_size`` episodes (separated_buffer.py:39-42)."""
        if not self.can_sample():
            return
        if self.use_linear_lr_decay:
            self.lr_decay(t_env, self.t_max)
        lib, st = _lib.lib, _lib.stream()
        s = self.store
        A, Bf, T1, F = self.n_agents, self.buffer_size, self.T1, self.F
        Fp = s["X"].shape[-1]
        rows = Bf * T1
        T = T1 - 1
        dist = parallel.dist_or_none() if self.use_dist else None
        world = dist.get_world_size() if dist else 1
        rank = dist.get_rank() if dist else 0
        # first batch_size (global) episodes are trained on (generate_data :371-394)
        n_train_global = self.batch_size
        n_train = parallel.shard_train_episodes(rank, world, Bf, n_train_global)
        # per-row loss gradients are O(1 / sum(alive)) ~ 1 / (rows trained on): scale them by the next
        # power of two so the split-f16 tensor-core products of the backward see O(1) operands
        self.grad_scale = float(2 ** max(0, math.ceil(math.log2(max(1, n_train_global * T)))))
        w = self._work_buffers(A, rows, Fp)
        actor, critic = self.stacks["actor"].flat, self.stacks["critic"].flat
        X = s["X"]
        R = self.args.rnn_hidden_dim
        ctx = self._ctx(w, s, A, Bf, T1, n_train, actor, critic, s["rnn_a"], s["rnn_c"], s["rnn_a"].stride(0), R,
                        s["actions"], s["avail"], F)

        # ---- once per train(): input LayerNorm statistics, pre-update values / log-probs, GAE
        _lib.check(lib.iplan_learner_row_stats(_lib.ptr(X), X.stride(0), Fp, F, rows, A, _lib.ptr(w["stat"]), st), "row_stats")
        assert X.is_contiguous()
        _lib.check(lib.iplan_learner_x_split(_lib.ptr(X), X.numel(), _lib.ptr(w["Xh"]), _lib.ptr(w["Xl"]), st), "x_split")
        self._forward(w, ctx, X, A, rows, Fp, F, actor, critic, train=False)
        w["old_logp"] = w["logp"].clone()
        w["old_value"] = w["value"].clone()
        _lib.check(lib.iplan_learner_gae(_lib.ptr(w["old_value"]), _lib.ptr(s["reward"]), _lib.ptr(s["alive"]),
                                         self.gamma, self.gae_lambda, T1, Bf, n_train, A,
                                         _lib.ptr(w["returns"]), _lib.ptr(w["adv"]), _lib.ptr(w["moments"]), st), "gae")
        if dist:
            dist.all_reduce(w["moments"])
        _lib.check(lib.iplan_learner_adv_finalize(_lib.ptr(w["moments"]), float(n_train_global * T), _lib.ptr(w["norm"]), A, st),
                   "adv_finalize")
        ctx = self._ctx(w, s, A, Bf, T1, n_train, actor, critic, s["rnn_a"], s["rnn_c"], s["rnn_a"].stride(0), R,
                        s["actions"], s["avail"], F)
        if self.keep_pre:
            mean, istd = w["norm"][:, 0:1], w["norm"][:, 1:2]
            self.last_pre = dict(values_all=w["old_value"].view(A, Bf, T1).clone(), returns=w["returns"].view(A, Bf, T1)[..., :T].clone(),
                                 advantages=((w["adv"] - mean) * istd).view(A, Bf, T1)[..., :T].clone(),
                                 old_logp=w["old_logp"].view(A, Bf, T1)[..., :T].clone())

        # ---- PPO epochs ------------------------------------------------------------------
        w["stats"].zero_()
        ga, gc = w["grads"]["actor"], w["grads"]["critic"]
        for _ in range(self.ppo_epoch):
            ga.zero_(); gc.zero_(); w["SM"].zero_()
            self._forward(w, ctx, X, A, rows, Fp, F, actor, critic, train=True)
            self._mark("fc1_bwd")
            _lib.check(lib.iplan_learner_fc1_backward(
                _lib.ptr(actor), self.stacks["actor"].stride(), _lib.ptr(critic), self.stacks["critic"].stride(),
                _lib.ptr(ga), _lib.ptr(gc), _lib.ptr(w["Xh"]), _lib.ptr(w["Xl"]), w["Xh"].stride(0), Fp, F, rows, A,
                _lib.ptr(w["Z1"]), _lib.ptr(w["Dh"]), _lib.ptr(w["Dl"]), _lib.ptr(w["gscale"]),
                _lib.ptr(w["SM"]), _lib.ptr(w["G"]), st), "fc1_backward")
            self._mark("allreduce")
            if dist:
                self.bucket.allreduce([ga, gc])      # ONE NCCL all-reduce per PPO epoch
            self._mark("adam")
            if self.keep_pre and _ == 0:
                self.first_grads = {"actor": ga / self.grad_scale, "critic": gc / self.grad_scale}
            for kind, g, col in (("actor", ga, 4), ("critic", gc, 5)):
                self.steps[kind] += 1
                stack = self.stacks[kind]
                _lib.check(lib.iplan_learner_adam(
                    _lib.ptr(stack.flat), _lib.ptr(g), _lib.ptr(self.exp_avg[kind]), _lib.ptr(self.exp_avg_sq[kind]),
                    _lib.ptr(self.masks[kind]), _lib.ptr(w["sq"]), stack.stride(), stack.total, A,
                    self.lrs[kind], 0.9, 0.999, self.optim_eps, self.steps[kind], self.max_grad_norm,
                    self.grad_scale, _lib.ptr(w["stats"]), col, st), "adam")

        self._mark("end")
        # ---- statistics: one device->host read per train() ---------------------------------
        stats = w["stats"].clone()
        if dist:
            part = stats[:, :4].contiguous()
            dist.all_reduce(part)
            stats[:, :4] = part
        tot = stats.sum(0).cpu() / float(self.ppo_epoch * self.num_mini_batch_ * A)
        self.train_info = dict(policy_loss=float(tot[0]), value_loss=float(tot[1]), dist_entropy=float(tot[2]),
                               ratio=float(tot[3]), actor_grad_norm=float(tot[4]), critic_grad_norm=float(tot[5]))
        self.count = 0                                      # clear_buffer (:312)
        if self.logger is not None and t_env - self.log_stats_t >= self.args.learner_log_interval:
            for k in ("value_loss", "policy_loss", "dist_entropy", "actor_grad_norm", "critic_grad_norm", "ratio"):
                self.logger.log_stat(self.log_prefix + k, self.train_info[k], t_env)

    num_mini_batch_ = 1

    # ---- reference-named helper (reference :344-365) ------------------------------------
    def compute_returns(self, agent_id, obs_all, rewards, terminated, rnn_state_critic_all):
        """obs_all [Bf,T+1,F], rewards [Bf,T,1], terminated (alive mask) [Bf,T+1,1] -> [Bf,T,1]."""
        v = self.mac.get_value_ippo(agent_id, obs_all, rnn_state_critic_all)[..., 0].contiguous()
        Bf, T1 = v.shape
        rew = th.zeros(Bf, T1, device=self.device)
        rew[:, :T1 - 1] = rewards.to(self.device)[..., 0]
        alive = terminated.to(self.device)[..., 0].float().contiguous()
        ret, adv = th.empty(Bf, T1, device=self.device), th.empty(Bf, T1, device=self.device)
        mom = th.zeros(1, 4, dtype=th.float64, device=self.device)
        _lib.check(_lib.lib.iplan_learner_gae(_lib.ptr(v), _lib.ptr(rew), _lib.ptr(alive), self.gamma, self.gae_lambda,
                                              T1, Bf, Bf, 1, _lib.ptr(ret), _lib.ptr(adv), _lib.ptr(mom), _lib.stream()), "gae")
        return ret[:, :T1 - 1].unsqueeze(-1)

    # ---- checkpoints (reference :319-341) -------------------------------------------------
    def save_models(self, path):
        self.mac.save_models(path)
        for i in range(self.n_agents):
            th.save(self.actor_optimizers[i].state_dict(), "{}/actor_{}_opt.th".format(path, i))
            th.save(self.critic_optimizers[i].state_dict(), "{}/critic_{}_opt.th".format(path, i))

    def load_models(self, paths, load_optimisers=False):
        self.mac.load_models(paths)
        if load_optimisers:
            if len(paths) == 1:
                paths = [copy.copy(paths[0]) for _ in range(self.n_agents)]
            for i in range(self.n_agents):
                self.actor_optimizers[i].load_state_dict(th.load("{}/actor_{}_opt.th".format(paths[i], i), map_location="cpu", weights_only=False))
                self.critic_optimizers[i].load_state_dict(th.load("{}/critic_{}_opt.th".format(paths[i], i), map_location="cpu", weights_only=False))


def eval_rows(mac, agent_id, obs, rnn_states, net, action=None, avail=None):
    """Forward one agent's actor/critic over arbitrary rows ``obs [..., F]`` with stored hidden
    inputs ``rnn_states [..., 64]`` (DcntrlMAC.get_value_ippo / eval_action_ippo, reference
    controllers/dcntrl_controller.py:61-85).  Returns (values [rows], logp [rows], entropy mean)."""
    dev = mac.device
    F = mac.input_shape
    x = obs.reshape(-1, F).to(dev, th.float32)
    rows = x.shape[0]
    Fp = (F + 31) // 32 * 32
    X = th.zeros(1, rows, Fp, device=dev)
    X[0, :, :F] = x
    h = rnn_states.reshape(-1, 64).to(dev, th.float32).contiguous()
    z = lambda *s, **k: th.zeros(*s, device=dev, **k)
    hz = lambda *s: th.zeros(*s, device=dev, dtype=th.float16)
    w = dict(stat=z(1, rows, 2), Wh=hz(1, 128, Fp), Wl=hz(1, 128, Fp), Xh=hz(1, rows, Fp), Xl=hz(1, rows, Fp),
             ws=z(1, 128), cc=z(1, 128), Z1=z(1, rows, 128),
             A1=z(1, 2, rows, 64), Z2=z(1, 2, rows, 64), A2=z(1, 2, rows, 64), GI=z(1, 2, rows, 192), GH=z(1, 2, rows, 192),
             logp=z(1, rows), ent=z(1, rows), value=z(1, rows))
    actor = mac.actor_stack.flat[agent_id:agent_id + 1]
    critic = mac.critic_stack.flat[agent_id:agent_id + 1]
    act = (action.reshape(-1).to(dev).to(th.int32) if action is not None else th.zeros(rows, dtype=th.int32, device=dev)).contiguous()
    av = (avail.reshape(rows, -1).to(dev) != 0).to(th.uint8).contiguous() if avail is not None else None
    lib, st, P = _lib.lib, _lib.stream(), _lib.ptr
    _lib.check(lib.iplan_learner_row_stats(P(X), X.stride(0), Fp, F, rows, 1, P(w["stat"]), st), "row_stats")
    _lib.check(lib.iplan_learner_x_split(P(X), X.numel(), P(w["Xh"]), P(w["Xl"]), st), "x_split")
    _lib.check(lib.iplan_learner_fc1_forward(P(actor), mac.actor_stack.stride(), P(critic), mac.critic_stack.stride(),
                                             P(w["Xh"]), P(w["Xl"]), w["Xh"].stride(0), Fp, F, rows, 1, P(w["stat"]),
                                             P(w["Wh"]), P(w["Wl"]), P(w["ws"]), P(w["cc"]), P(w["Z1"]), st), "fc1_forward")
    c = _lib.LearnerCtx()
    c.actor, c.critic = P(actor), P(critic)
    c.actor_stride, c.critic_stride = mac.actor_stack.stride(), mac.critic_stack.stride()
    c.feat_dim, c.n_actions, c.n_agents, c.T1, c.n_eps, c.n_train_eps = F, mac.args.n_actions, 1, 1, rows, 0
    # one hidden array per net type: the unused one just needs to be readable
    c.rnn_a, c.rnn_c, c.rnn_stride_agent, c.rnn_ld = P(h), P(h), 0, 64
    c.actions, c.avail = P(act), P(av)
    for k in ("Z1", "A1", "Z2", "A2", "GI", "GH"):
        setattr(c, k, P(w[k]))
    c.stat = P(w["stat"])
    c.logp_out, c.ent_out, c.value_out = P(w["logp"]), P(w["ent"]), P(w["value"])
    import ctypes
    _lib.check(lib.iplan_learner_tail(ctypes.byref(c), 0, st), "learner_tail")
    return w["value"][0], w["logp"][0], w["ent"][0].mean()
