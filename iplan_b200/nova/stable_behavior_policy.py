"""Behavioural-incentive module (soft-update variant = iPLAN) — host-side mirror of the
reference's ``Behavior_policy`` (/root/reference/nova/stable_behavior_policy.py:13-123) for
the rollout entry point ``latent_update``; the arithmetic is kernel K1b
(csrc/behavior_step.cu).

Same constructor, same ``latent_update(history, encoder_hidden, prev_latent) ->
(np latent [B,A,N,L], torch hidden [B,1,A,N,E])`` contract (the reference returns the
hidden state as a torch tensor and accepts numpy on the first call / a tensor
afterwards, :101-121), same ``behavior_encoder[i]`` state_dict keys and
``behavior_encoder_{i}.th`` files.  The auxiliary reconstruction learner (``learn``, reference :161-279, SURVEY §8f
rank 3): kernel csrc/beh_learn.cu (the pinned oracle oracle/iplan_oracle.py::behavior_learn_agent line by line), checked
against the reference's recorded ``learn`` call (tools/check_beh_learn.py, tests/test_gpu_learner.py): losses 2e-7,
every gradient tensor <= 1e-5 relative, post-step weights 1.5e-8.  It is a plain-FFMA first version (estimated seconds
per call at 512 envs; the tensor-core version is future work); ``behavior_optimizer_{i}_opt.th`` holds the Adam state in
torch.optim.Adam's state_dict format.
"""
import copy
import os

import numpy as np
import torch

from .. import _lib
from ..modules.flat import ParamStack


class _BehAdam:
    """torch.optim.Adam-compatible ``state_dict`` of one agent's (encoder + decoder) optimiser (reference :59-62, files
    ``behavior_optimizer_{i}_opt.th`` :288): parameter ids run over the encoder tensors, then the decoder tensors."""

    def __init__(self, owner, index):
        self.owner, self.index = owner, index

    def _entries(self):
        o, out, pid = self.owner, [], 0
        for kind, stack in (("enc", o.stack), ("dec", o.dec_stack)):
            for (name, shape), off in zip(stack.spec, stack.offsets):
                n = 1
                for d in shape:
                    n *= d
                out.append((pid, kind, shape, off, n))
                pid += 1
        return out

    def state_dict(self):
        o = self.owner
        w, st = o._learn_state(), {}
        for pid, kind, shape, off, n in self._entries():
            if w["step"] == 0:
                continue
            st[pid] = {"step": torch.tensor(float(w["step"])),
                       "exp_avg": w["m_" + kind][self.index, off:off + n].view(shape).detach().cpu().clone(),
                       "exp_avg_sq": w["v_" + kind][self.index, off:off + n].view(shape).detach().cpu().clone()}
        group = {"lr": float(o.args.lr_behavior), "betas": (0.9, 0.999), "eps": float(o.args.optim_eps),
                 "weight_decay": float(getattr(o.args, "weight_decay", 0)), "amsgrad": False, "maximize": False, "foreach": None,
                 "capturable": False, "differentiable": False, "fused": None, "params": [e[0] for e in self._entries()]}
        return {"state": st, "param_groups": [group]}

    def load_state_dict(self, sd):
        o = self.owner
        w = o._learn_state()
        for pid, kind, shape, off, n in self._entries():
            if pid in sd["state"]:
                s_ = sd["state"][pid]
                w["m_" + kind][self.index, off:off + n] = s_["exp_avg"].reshape(-1).to(o.device)
                w["v_" + kind][self.index, off:off + n] = s_["exp_avg_sq"].reshape(-1).to(o.device)
                w["step"] = int(s_["step"])


class Behavior_policy:
    def __init__(self, args, logger=None):
        self.device = torch.device("cuda" if args.use_cuda else "cpu")
        if self.device.type != "cuda":
            raise RuntimeError("iplan_b200.Behavior_policy runs on CUDA only (no CPU path); set args.use_cuda=True")
        self.args = args
        self.logger = logger
        self.n_agents = args.n_agents
        self.max_vehicle_num = args.max_vehicle_num
        self.max_history_len = args.max_history_len
        self.latent_dim = args.latent_dim
        self.soft_update_coef = args.soft_update_coef
        self._build_nets(args)
        self.behavior_encoder = self.stack.nets
        self.behavior_decoder = self.dec_stack.nets
        self._stage = None        # device staging buffers of the pipelined numpy entry point
        self._learn = None          # Adam moments / work buffers of learn()
        self.learn_calls = 0
        self.seed = int(getattr(args, "seed", 112358))
        self.log_prefix = getattr(args, "log_prefix", "")
        self.log_stats_t = -getattr(args, "learner_log_interval", 0) - 1
        self.behavior_optimizer = [_BehAdam(self, i) for i in range(self.n_agents)]
        self.debug_keep = None      # uint8 [A, B, n_pos, N, W, 64] explicit dropout draw for the next learn() (parity runs)

    def _build_nets(self, args):
        """Parameter stacks of the encoder (``self.stack``) and of the reconstruction decoder (``self.dec_stack``)."""
        assert args.encoder_rnn_dim == 32 and args.num_encoder_layer == 1, "kernel K1b is built for E = 32, one layer"
        self.stack = ParamStack("beh", self.n_agents, (args.obs_shape_single, args.latent_dim), device=self.device)
        # the reconstruction decoder of the auxiliary learner (reference :48-53)
        self.dec_stack = ParamStack("bdec", self.n_agents, (args.obs_shape_single, args.latent_dim, args.decoder_rnn_dim), device=self.device)

    # ---- device path: tensors laid out [A, B, N, *] ----------------------------------
    def behavior_step(self, window, hid_io, lat_prev, lat_out, win_stride_step=0, win_pad=0):
        """window [A,B,N,W*o], hid_io [A,B,N,E] (in place), lat_prev/lat_out [A,B,N,L].
        With ``win_stride_step`` != 0 the window is read in place from a time-strided store: ``window`` is the [A,B,N,o]
        view of its oldest real row, later rows ``win_stride_step`` elements apart, ``win_pad`` leading rows are zeros."""
        A, B, N, _ = window.shape
        rc = _lib.lib.iplan_behavior_step_ex(
            _lib.ptr(self.stack.flat), self.stack.stride(),
            _lib.view(window), int(win_stride_step), int(win_pad), _lib.view(hid_io), _lib.view(lat_prev), _lib.view(lat_out),
            float(self.soft_update_coef), B, A, N, self.args.obs_shape_single, self.latent_dim,
            self.max_history_len, _lib.stream())
        _lib.check(rc, "behavior_step")
        return lat_out, hid_io

    # ---- reference-compatible entry point (reference :83-123) -------------------------
    def latent_update(self, history, encoder_hidden, prev_latent):
        dev = self.device
        hist_h = _lib.as_host(history)
        prev_dev = _lib.device_shadow(prev_latent)          # the latent this method returned last step: still on the device
        prev_h = None if prev_dev is not None else _lib.as_host(prev_latent)
        B, A, N, W, o = hist_h.shape
        if torch.is_tensor(encoder_hidden) and encoder_hidden.is_cuda:
            hid = encoder_hidden.detach().to(torch.float32).clone()
        else:
            hid = _lib.to_device(encoder_hidden)
        perm = (1, 0, 2, 3)
        if B >= _lib.PIPELINE_MIN_ROWS:
            # one native call (csrc/host_api.cu): copy-in, K1b and copy-out overlap piece by piece over the envs
            L = int(prev_latent.shape[-1])
            key = (B, A, N, W, o, L)
            if self._stage is None or self._stage[0] != key:
                self._stage = (key, torch.empty(B, A, N, W, o, device=dev), torch.empty(B, A, N, L, device=dev))
            _, hist, prev_stage = self._stage
            hist_h = hist_h.contiguous()
            _lib.io_bytes["h2d"] += hist_h.numel() * 4
            if prev_dev is not None:
                prev = prev_dev if prev_dev.dtype == torch.float32 and prev_dev.is_contiguous() else prev_dev.to(torch.float32).contiguous()
                _lib.io_bytes["h2d_saved"] += prev.numel() * prev.element_size()
            else:
                prev, prev_h = prev_stage, prev_h.contiguous()
                _lib.io_bytes["h2d"] += prev_h.numel() * 4
            assert hid.is_contiguous() and hid.numel() == B * A * N * self.args.encoder_rnn_dim, hid.shape
            new = torch.empty(B, A, N, L, device=dev)           # fresh: the shadow of the returned array
            new_h = torch.empty(B, A, N, L, dtype=torch.float32, pin_memory=True)
            _lib.check(_lib.lib.iplan_behavior_latent_update_host(
                _lib.ptr(self.stack.flat), self.stack.stride(), _lib.host_ptr(hist_h), _lib.ptr(hist), _lib.host_ptr(prev_h), _lib.ptr(prev),
                _lib.ptr(hid), _lib.ptr(new), _lib.host_ptr(new_h), float(self.soft_update_coef),
                B, A, N, o, L, W, min(8, _lib.MAX_PIPELINE_CHUNKS), _lib.stream()), "behavior_latent_update_host")
            _lib.io_bytes["d2h"] += new.numel() * 4
            return _lib.adopt_host(new_h, new), hid
        hist = _lib.to_device(hist_h)
        prev = _lib.to_device(prev_latent)
        new = torch.empty_like(prev)
        hid_v = hid[:, 0].permute(perm)                          # [B,1,A,N,E] -> [A,B,N,E] view
        self.behavior_step(hist.reshape(B, A, N, W * o).permute(perm), hid_v,
                           prev.permute(perm), new.permute(perm))
        return _lib.to_host(new, shadow=True), hid

    def _learn_state(self):
        """Optimiser state (Adam moments with the parameter buffers' layout) and work buffers of ``learn``."""
        if self._learn is None:
            dev, A = self.device, self.n_agents
            z = lambda t: torch.zeros_like(t)
            self._learn = dict(g_enc=z(self.stack.flat), g_dec=z(self.dec_stack.flat), m_enc=z(self.stack.flat), v_enc=z(self.stack.flat),
                               m_dec=z(self.dec_stack.flat), v_dec=z(self.dec_stack.flat),
                               ones_enc=torch.ones(self.stack.total, device=dev), ones_dec=torch.ones(self.dec_stack.total, device=dev),
                               sq=torch.zeros(A, device=dev), stats=torch.zeros(A, 8, device=dev), step=0, scratch=None)
        return self._learn

    def learn(self, batch, t_env):
        """Reference :161-279: for every agent-net, walk the T-1-W window positions of every episode with the decoder and
        the encoder (hidden states and the soft-updated latent carried across positions), masked L1 reconstruction of the
        next window (:226-233), one backward through everything, separate gradient clipping of encoder and decoder
        (:248-256), one Adam step (:258).  Returns (behavior_loss, stability_loss, total_loss) lists of per-agent values."""
        args, dev = self.args, self.device
        if float(getattr(args, "behavior_variation_penalty", 0)) != 0.0:
            raise NotImplementedError("only behavior_variation_penalty = 0 (the iPLAN setting) is built: the stability term is reported, not differentiated")
        A, N, o, L, W = self.n_agents, self.max_vehicle_num, args.obs_shape_single, self.latent_dim, self.max_history_len
        hist = batch["history"][:, :-1]                                  # [B, T, A, N, o]
        term = batch["terminated"][:, :-1, :, 0].to(torch.float32)      # [B, T, A]
        mask = (1.0 - term) if args.env == "MPE" else term               # :186-189
        B, T = hist.shape[0], hist.shape[1]
        n_pos = T - 1 - W
        hist_a = hist.permute(2, 0, 1, 3, 4).contiguous()
        mask_a = mask.permute(2, 0, 1).contiguous()                      # [A, B, T]
        cs = torch.cumsum(mask_a.sum(dim=1), dim=1)                      # [A, T]
        j = torch.arange(n_pos, device=dev)
        msum = (cs[:, j + W] - cs[:, j]) * (N * o)                       # unmasked elements of the next-window at position j
        scale = ((o * N) / (msum + 1e-10) / n_pos).contiguous()
        bl, sl, norms = self._learn_step(hist_a, mask_a, scale, n_pos)
        behavior_loss = [np.asarray(float(bl[i]), dtype=np.float32) for i in range(A)]
        stability_loss = [np.asarray(float(sl[i]), dtype=np.float32) for i in range(A)]
        total_loss = [np.asarray(float(bl[i]), dtype=np.float32) for i in range(A)]          # penalty = 0
        self._log(t_env, dict(behavior_loss=float(bl.sum()), stability_loss=float(sl.sum()), behavior_total=float(bl.sum()),
                              behavior_encoder_grad_norm=float(norms[:, 0].sum()), behavior_decoder_grad_norm=float(norms[:, 1].sum())))
        return behavior_loss, stability_loss, total_loss

    def _learn_step(self, hist_a, mask_a, scale, n_pos, windows=None):
        """Loss and gradients of every agent-net (one native call), then per agent-net the separately clipped encoder and
        decoder gradients and one Adam step over both.  hist_a [A,B,T,N,o], mask_a [A,B,T] (read at the target row),
        scale [A,n_pos].  ``windows = (win_step, win_first)`` selects a window geometry (iplan_beh_learn_windows); None is
        the soft update's sliding window (iplan_beh_learn).  Returns (behavior loss [A], stability loss [A], clip norms
        [A,8]: column 0 encoder, 1 decoder) on the host."""
        args, dev = self.args, self.device
        A, N, o, L, W = self.n_agents, self.max_vehicle_num, args.obs_shape_single, self.latent_dim, self.max_history_len
        B, T = hist_a.shape[1], hist_a.shape[2]
        lib, st, ptr = _lib.lib, _lib.stream(), _lib.ptr
        w = self._learn_state()
        scratch_floats = lib.iplan_beh_learn_scratch_floats if windows is None else lib.iplan_beh_learn_tile_scratch_floats
        need = scratch_floats(A, B, n_pos, N, o, L, W)
        if w["scratch"] is None or w["scratch"].numel() < need:
            w["scratch"] = torch.empty(need, device=dev)
        w["g_enc"].zero_(); w["g_dec"].zero_(); w["stats"].zero_()
        b_loss, s_loss = torch.zeros(A, device=dev), torch.zeros(A, device=dev)
        keep = self.debug_keep
        self.debug_keep = None
        if keep is not None:
            keep = keep.to(dev, torch.uint8).contiguous()
            assert tuple(keep.shape) == (A, B, n_pos, N, W, args.decoder_rnn_dim), keep.shape
        common = (ptr(self.stack.flat), self.stack.stride(), ptr(self.dec_stack.flat), self.dec_stack.stride(), ptr(w["g_enc"]), ptr(w["g_dec"]),
                  ptr(hist_a), ptr(mask_a), ptr(scale), ptr(keep), ptr(b_loss), ptr(s_loss), ptr(w["scratch"]), w["scratch"].numel(),
                  self.seed, self.learn_calls, float(args.decoder_dropout), float(self.soft_update_coef), float(args.thres_small_variation),
                  A, B, T, N, o, L, W)
        if windows is None:
            _lib.check(lib.iplan_beh_learn(*common, st), "beh_learn")
        else:
            _lib.check(lib.iplan_beh_learn_windows(*common, n_pos, int(windows[0]), int(windows[1]), st), "beh_learn_windows")
        self.learn_calls += 1
        self._adam_step()
        return b_loss.cpu(), s_loss.cpu(), w["stats"].cpu()

    def _adam_step(self):
        """After a learn kernel has filled g_enc / g_dec: keep the raw gradients in ``last_grads`` (parity checks), then
        per agent-net clip the encoder and decoder gradients separately to max_grad_norm (pre-clip norms into stats
        columns 0 and 1) and take one Adam step (lr_behavior) over both."""
        args, w = self.args, self._learn_state()
        lib, st, ptr, A = _lib.lib, _lib.stream(), _lib.ptr, self.n_agents
        self.last_grads = dict(enc=w["g_enc"].clone(), dec=w["g_dec"].clone())       # raw (unclipped) gradients, for parity checks
        w["step"] += 1
        for stack, g, m, v, ones, col in ((self.stack, w["g_enc"], w["m_enc"], w["v_enc"], w["ones_enc"], 0),
                                          (self.dec_stack, w["g_dec"], w["m_dec"], w["v_dec"], w["ones_dec"], 1)):
            _lib.check(lib.iplan_learner_adam(ptr(stack.flat), ptr(g), ptr(m), ptr(v), ptr(ones), ptr(w["sq"]), stack.stride(),
                                              stack.total, A, float(args.lr_behavior), 0.9, 0.999, float(args.optim_eps), w["step"],
                                              float(args.max_grad_norm), 1.0, ptr(w["stats"]), col, st), "adam")

    def _log(self, t_env, train_info):
        self.train_info = train_info
        if self.logger is not None and t_env - self.log_stats_t >= getattr(self.args, "learner_log_interval", 0):
            for k, v in self.train_info.items():
                self.logger.log_stat(self.log_prefix + k, v, t_env)

    # ---- checkpoints (reference :282-312) -------------------------------------------
    def save_models(self, path):
        for i, net in enumerate(self.behavior_encoder):
            torch.save({k: v.detach().cpu() for k, v in net.state_dict().items()}, f"{path}/behavior_encoder_{i}.th")
        for i, net in enumerate(self.behavior_decoder):
            torch.save({k: v.detach().cpu() for k, v in net.state_dict().items()}, f"{path}/behavior_decoder_{i}.th")
        for i in range(self.n_agents):
            torch.save(self.behavior_optimizer[i].state_dict(), "{}/behavior_optimizer_{}_opt.th".format(path, i))

    def load_models(self, paths, load_optimisers=False):
        if len(paths) == 1:
            paths = [copy.copy(paths[0]) for _ in range(self.n_agents)]
        for i, net in enumerate(self.behavior_encoder):
            net.load_state_dict(torch.load(os.path.join(paths[i], f"behavior_encoder_{i}.th"),
                                           map_location="cpu", weights_only=False))
        for i, net in enumerate(self.behavior_decoder):
            f = os.path.join(paths[i], f"behavior_decoder_{i}.th")
            if os.path.exists(f):
                net.load_state_dict(torch.load(f, map_location="cpu", weights_only=False))
        if load_optimisers:
            for i in range(self.n_agents):
                self.behavior_optimizer[i].load_state_dict(torch.load("{}/behavior_optimizer_{}_opt.th".format(paths[i], i),
                                                                      map_location="cpu", weights_only=False))
