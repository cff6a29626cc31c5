"""Rollout runner on synthetic Heterogeneous-Highway-shaped observations.

Mirrors the reference's ``ParallelRunner`` (/root/reference/runners/ippo_parallel_runner.py:7-287):
same ``ParallelRunner(args, env, logger)`` / ``setup(scheme, groups, preprocess, mac,
behavior_learner, prediction_learner)`` / ``run(test_mode) -> (EpisodeBatch, avg_win,
avg_rwd, avg_len)`` / ``get_env_info`` / ``close_env`` / ``t_env`` surface, and the same
per-timestep order (reference :166-266):

    select_actions(t) -> env.step -> GAT update(history_{t+1}, att_t, beh_t)
                      -> behaviour update(window_{t+1}, beh_t) -> store pre-transition t+1

The simulator, the subprocess env vector and the Python observation wrapper are out of
scope (SURVEY §2 rows 21-24): ``SyntheticHighway`` generates what they would hand to the
runner, in the shapes and value ranges SURVEY §8d fixes.

Two paths through the same kernels:
 * ``run()`` — device resident: K1 / K1b / K1c read and write the packed EpisodeBatch
   directly (no host round trip per step);
 * ``run_reference_api()`` — the reference's call pattern: numpy arrays into
   ``GAT_latent_update`` / ``latent_update`` / ``EpisodeBatch.update`` /
   ``select_actions_ippo`` every step (bench.py's e2e leg).
"""
from functools import partial
from types import SimpleNamespace

import numpy as np
import torch as th

from .. import _lib
from ..components.episode_buffer import EpisodeBatch
from ..components.transforms import OneHot


class SyntheticHighway:
    """Seeded stand-in for SubprocVecEnv + observation wrapper.  Per episode it holds, on the
    device, ``history[t]`` [B,A,N,o] for t = 0..T (col 0 presence = 1, other columns
    U(-1,1), slots >= K_t exactly 0 with K_t = min(N, n_obs + t//3)), rewards ~ N(0,1) and
    per-agent ``terminated`` flags that latch with a per-step hazard (0.002 "mild", 0.01
    "chaotic").  The 10-step window is the last W single histories, zero padded in front
    (observation_wrapper.py:101-119)."""

    def __init__(self, args, n_envs, hazard=0.01, seed=112358, device="cuda"):
        self.args, self.B, self.hazard, self.seed, self.device = args, n_envs, hazard, seed, device
        self.A, self.N, self.o = args.n_agents, args.max_vehicle_num, args.obs_shape_single
        self.T, self.W = args.episode_limit, args.max_history_len
        self.n_obs = getattr(args, "n_obs_vehicles", self.N)
        self.episodes = 0
        self.generate()

    def generate(self):
        g = th.Generator(device=self.device)
        g.manual_seed(self.seed + 7919 * self.episodes)
        B, A, N, o, T = self.B, self.A, self.N, self.o, self.T
        h = th.rand(T + 1, B, A, N, o, device=self.device, generator=g) * 2 - 1
        h[..., 0] = 1.0
        for t in range(T + 1):
            k = min(N, self.n_obs + t // 3)
            h[t, :, :, k:] = 0.0
        self.history = h
        self.reward = th.randn(T, B, A, device=self.device, generator=g)
        dies = th.rand(T, B, A, device=self.device, generator=g) < self.hazard
        self.terminated = (th.cumsum(dies.int(), dim=0) > 0)
        self.episodes += 1

    def window(self, t):
        """[B,A,N,W,o]: single histories t-W+1 .. t, zeros before the episode start."""
        B, A, N, o, W = self.B, self.A, self.N, self.o, self.W
        w = th.zeros(B, A, N, W, o, device=self.device)
        lo = max(0, t - W + 1)
        w[:, :, :, W - (t - lo + 1):] = self.history[lo:t + 1].permute(1, 2, 3, 0, 4)
        return w

    def host_episode(self):
        """Host-memory copies of the episode (numpy, fp32), as a CPU simulator + observation wrapper
        would deliver them: history[t] [B,A,N,o], window[t] [B,A,N,W,o], reward [T,B,A],
        terminated [T,B,A], in page-locked memory.  Built once per generated episode (2.6 GB at B=512)."""
        if getattr(self, "_host", None) is None or self._host["episode"] != self.episodes:
            T = self.T
            self._host = dict(episode=self.episodes,
                              history=[_lib.pinned_numpy(self.history[t]) for t in range(T + 1)],
                              window=[_lib.pinned_numpy(self.window(t)) for t in range(T + 1)],
                              reward=_lib.pinned_numpy(self.reward), terminated=_lib.pinned_numpy(self.terminated))
        return self._host

    def close(self):
        pass


def make_scheme(args):
    """The scheme run_sequential builds (run_ippo.py:160-184)."""
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


class ParallelRunner:
    def __init__(self, args, env, logger):
        self.args, self.env, self.logger = args, env, logger
        self.batch_size = args.batch_size_run
        self.episode_limit = args.episode_limit
        self.n_agents = args.n_agents
        self.max_vehicle_num = args.max_vehicle_num
        self.t = 0
        self.t_env = 0
        self.batch = None

    def setup(self, scheme, groups, preprocess, mac, behavior_learner, prediction_learner):
        self.new_batch = partial(EpisodeBatch, scheme, groups, self.batch_size, self.episode_limit + 1,
                                 preprocess=preprocess, device=self.args.device)
        self.mac, self.scheme, self.groups, self.preprocess = mac, scheme, groups, preprocess
        self.behavior_learner, self.prediction_learner = behavior_learner, prediction_learner

    def get_env_info(self, args):
        return {"n_agents": self.n_agents, "n_actions": args.n_actions,
                "state_shape": args.obs_shape_single * self.max_vehicle_num,
                "episode_limit": self.episode_limit,
                "obs_shape": args.obs_shape_single * getattr(args, "n_obs_vehicles", self.max_vehicle_num)}

    def close_env(self):
        self.env.close()

    # ---- episode storage: one packed batch, recycled ------------------------------------
    def _fresh_batch(self):
        if self.batch is None:
            self.batch = self.new_batch()
            return self.batch
        b = self.batch
        d = b.packed_dims
        b.packed.zero_()
        b.packed[..., d.col_id:d.col_id + d.A] = th.eye(d.A, device=b.packed.device).view(d.A, 1, 1, d.A)
        for k, v in b.data.transition_data.items():
            if k not in ("history", "attention_latent", "behavior_latent"):
                v.zero_()
        return b

    # ---- device-resident episode ------------------------------------------------------------
    def run(self, test_mode=False):
        env, args = self.env, self.args
        B, A, N, T = self.batch_size, self.n_agents, self.max_vehicle_num, self.episode_limit
        W, o, E = args.max_history_len, args.obs_shape_single, args.encoder_rnn_dim
        batch = self._fresh_batch()
        d = batch.packed_dims
        dev = batch.packed.device
        packed = batch.packed                                           # [A,B,T+1,Fp]
        slots = packed[..., :N * d.S].view(A, B, T + 1, N, d.S)
        hist_v, att_v, beh_v = slots[..., :o], slots[..., o:o + d.D], slots[..., o + d.D:]
        rnn_a = batch["rnn_states_actors"].permute(2, 0, 1, 3)         # [A,B,T+1,R] views
        rnn_c = batch["rnn_states_critics"].permute(2, 0, 1, 3)
        batch["avail_actions"].fill_(1)
        batch["filled"].fill_(1)
        enc_hid = th.zeros(A, B, N, E, device=dev)
        zeros_att = th.zeros(A, B, N, d.D, device=dev)
        zeros_beh = th.zeros(A, B, N, d.L, device=dev)
        # per-episode output buffers of K1c: [T+1][A][B], one contiguous [A][B] plane per timestep (no alloc / copy per step)
        actions_steps = th.zeros(T + 1, A, B, dtype=th.int32, device=dev)
        logp_steps = th.empty(T, A, B, device=dev)
        value_steps = th.empty(T, A, B, device=dev)
        onehot_cols = packed[..., d.col_act:d.col_act + d.n_actions]    # [A,B,T+1,n_act] view
        # The synthetic simulator holds the whole episode's observations in HBM: they enter the episode store in ONE
        # strided device copy (a live simulator would write row t each step through observation_wrapper.step()).  K1 reads
        # row t, K1b reads its W-step window in place from rows t-W+1..t of the store: no shifted window copy per step.
        hist_v.copy_(env.history.permute(2, 1, 0, 3, 4))
        # K1b's window rows come from the simulator's dense history [T+1,B,A,N,o] (what the observation wrapper's device window
        # is): 20 contiguous bytes per slot and row next to its neighbours', instead of 20 of every 180 bytes of the packed store
        # (ncu: 227 MB of DRAM reads per launch for 28 MB of window)
        hist_src = env.history.permute(0, 2, 1, 3, 4)                   # [T+1,A,B,N,o] view
        hist_step = env.history.stride(0)

        events = getattr(self, "gat_events", None)
        noise = getattr(self, "noise_hook", None)      # parity tests: noise(kind, index) -> explicit noise tensor or None

        def timed(tag, fn, *a, **k):
            """Kernel launch, optionally bracketed by CUDA events on the launching stream (bench.py)."""
            if events is None:
                return fn(*a, **k)
            e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            events.append((tag, e0, e1))
            return out

        gat_calls = [0]

        def gat(*a):
            gum = noise("gumbel", gat_calls[0]) if noise is not None else None      # [A,B,N,N-1,2] or None (Philox)
            gat_calls[0] += 1
            if events is None:
                return self.prediction_learner.gat_step(*a, gumbel=gum)
            ev = [th.cuda.Event(enable_timing=True) for _ in range(3)]
            for e in ev:
                e.record()                   # creates the handles; the library re-records them around its two kernels
            out = self.prediction_learner.gat_step(*a, gumbel=gum, events=ev)
            events.append(("gat_recur", ev[0], ev[1]))
            events.append(("gat_attend", ev[1], ev[2]))
            events.append(("gat", ev[0], ev[2]))
            return out

        gat(hist_v[:, :, 0], zeros_beh, zeros_att, att_v[:, :, 0])
        for t in range(T):
            timed("ctrl", self.mac.controller_step,
                  packed[:, :, t], rnn_a[:, :, t], rnn_c[:, :, t], rnn_a[:, :, t + 1], rnn_c[:, :, t + 1],
                  None, test_mode=test_mode, uniforms=noise("uniforms", t) if noise is not None else None,
                  next_onehot=onehot_cols[:, :, t + 1], this_onehot=onehot_cols[:, :, 0] if t == 0 else None,
                  out=(actions_steps[t], logp_steps[t], value_steps[t]))
            gat(hist_v[:, :, t + 1], beh_v[:, :, t], att_v[:, :, t], att_v[:, :, t + 1])
            first = max(0, t + 2 - W)                                   # oldest time inside the window of time t+1
            timed("beh", self.behavior_learner.behavior_step, hist_src[first], enc_hid, beh_v[:, :, t], beh_v[:, :, t + 1],
                  win_stride_step=hist_step, win_pad=max(0, W - (t + 2)))
        actions_all = actions_steps.permute(1, 2, 0)                    # [A,B,T+1]
        self.last_logp, self.last_values = logp_steps, value_steps      # [T,A,B] of the episode just run (parity tests)
        # episode-level stores in the reference's layout [B,T+1,A,*]
        batch["actions"][..., 0] = actions_all.permute(1, 2, 0).long()
        batch["actions_onehot"].zero_().scatter_(-1, batch["actions"], 1.0)
        batch["reward"][:, :T, :, 0] = env.reward.permute(1, 0, 2)
        batch["terminated"][:, :T, :, 0] = env.terminated.permute(1, 0, 2).to(th.uint8)
        self.t = T
        alive_envs = (~env.terminated.all(dim=2)).sum().item() if not test_mode else 0
        if not test_mode:
            self.t_env += B * T
        avg_rwd = float(env.reward.sum(dim=(0, 2)).mean())
        avg_len = float(alive_envs) / B
        if self.logger is not None:
            self._log(0.0, avg_rwd, avg_len)
        return batch, 0.0, avg_rwd, avg_len

    # ---- the reference's call pattern: numpy in / numpy out every step ---------------------------
    def run_reference_api(self, test_mode=False):
        env, args = self.env, self.args
        B, A, N, T = self.batch_size, self.n_agents, self.max_vehicle_num, self.episode_limit
        batch = self._fresh_batch()
        avail = np.ones((B, A, args.n_actions), dtype=np.int64)
        rnn_a = np.zeros((B, args.recurrent_N, A, args.rnn_hidden_dim), dtype=np.float32)
        rnn_c = np.zeros_like(rnn_a)
        enc_rnn = np.zeros((B, args.num_encoder_layer, A, N, args.encoder_rnn_dim), dtype=np.float32)
        beh = np.zeros((B, A, N, args.latent_dim), dtype=np.float32)
        att = np.zeros((B, A, N, args.attention_dim), dtype=np.float32)
        host = env.host_episode()                     # what the env / observation wrapper hand over (host memory)
        hist_np, win_np = host["history"], host["window"]
        single = hist_np[0]
        att = self.prediction_learner.GAT_latent_update(single, att, beh)
        batch.update({"avail_actions": avail, "rnn_states_actors": rnn_a, "rnn_states_critics": rnn_c,
                      "history": single, "behavior_latent": beh, "attention_latent": att}, ts=0)
        rew, term = host["reward"], host["terminated"]
        for t in range(T):
            _, actions, _, rnn_a, rnn_c = self.mac.select_actions_ippo(batch, t_ep=t, test_mode=test_mode)
            batch.update({"actions": actions}, ts=t, mark_filled=False)
            single = hist_np[t + 1]
            att = self.prediction_learner.GAT_latent_update(single, att, beh)
            beh, enc_rnn = self.behavior_learner.latent_update(win_np[t + 1], enc_rnn, beh)
            batch.update({"reward": rew[t], "terminated": term[t]}, ts=t, mark_filled=False)
            batch.update({"avail_actions": avail, "rnn_states_actors": rnn_a, "rnn_states_critics": rnn_c,
                          "history": single, "behavior_latent": beh, "attention_latent": att}, ts=t + 1, mark_filled=True)
        self.t = T
        if not test_mode:
            self.t_env += B * T
        return batch, 0.0, float(rew.sum(axis=(0, 2)).mean()), float(T)

    def _log(self, win_rates, episode_reward, episode_len):
        self.logger.log_stat(self.args.log_prefix + "Average episode_win_num", win_rates, self.t_env)
        self.logger.log_stat(self.args.log_prefix + "Average episode_reward", episode_reward, self.t_env)
        self.logger.log_stat(self.args.log_prefix + "Average episode_len", episode_len, self.t_env)


def build_system(n_envs, env="highway", hazard=0.01, seed=112358, logger=None, **overrides):
    """Wire args -> scheme -> MAC -> learner -> behaviour / prediction modules -> runner, as
    run_sequential does (run_ippo.py:122-225), on synthetic observations."""
    from ..config import make_args
    from ..controllers.dcntrl_controller import DcntrlMAC
    from ..learners.ippo_learner import IPPOLearner
    from ..nova.prediction_policy import Prediction_policy
    from ..nova import behavior_FC_policy, behavior_policy, stable_behavior_policy
    over = dict(batch_size_run=n_envs, buffer_size=n_envs, batch_size=n_envs - 1, use_cuda=True, device="cuda", seed=seed)
    if env != "highway" and "episode_limit" in overrides:
        overrides["episode_length"] = overrides.pop("episode_limit")
    over.update(overrides)
    args = make_args(env, **over)
    th.manual_seed(seed)
    scheme, groups, preprocess = make_scheme(args)
    sim = SyntheticHighway(args, n_envs, hazard=hazard, seed=seed)
    runner = ParallelRunner(args, sim, logger)
    probe = EpisodeBatch(scheme, groups, 1, 2, preprocess=preprocess, device="cpu")    # scheme incl. actions_onehot
    mac = DcntrlMAC(probe.scheme, groups, args)
    learner = IPPOLearner(mac, probe.scheme, logger, args)
    # behavior_fully_connected: True is the iPLAN-FC ablation and wins over soft_update_enable, whose False is the
    # iPLAN-Hard ablation (run_ippo.py:200-209)
    if args.behavior_fully_connected:
        behavior_module = behavior_FC_policy
    else:
        behavior_module = stable_behavior_policy if args.soft_update_enable else behavior_policy
    behavior = behavior_module.Behavior_policy(args, logger)
    prediction = Prediction_policy(args, logger)
    runner.setup(scheme, groups, preprocess, mac, behavior, prediction)

    def run_and_train(api=False):
        batch, *_ = (runner.run_reference_api() if api else runner.run())
        learner.insert_episode_batch(batch)
        learner.train(runner.t_env)
        return batch

    return SimpleNamespace(args=args, env=sim, runner=runner, mac=mac, learner=learner, behavior=behavior,
                           prediction=prediction, run_and_train=run_and_train, scheme=scheme, groups=groups,
                           preprocess=preprocess)
