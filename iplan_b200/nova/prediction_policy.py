"""Instant-incentive (GAT) module — host-side mirror of the reference's
``Prediction_policy`` (/root/reference/nova/prediction_policy.py:14-118) for the rollout
entry point ``GAT_latent_update``; the arithmetic is kernel K1 (csrc/gat_step.cu).

Same constructor, same ``GAT_latent_update(history_single, encoder_hidden,
behavior_latent) -> np.float32 [B, A, N, D]`` contract, same ``pred_GAT[i]`` modules
(state_dict keys/shapes) and ``pred_GAT_{i}.th`` checkpoint files.  The auxiliary
trajectory-prediction learner (``learn``, reference :168-253) is a "next" row of the scope table
(SURVEY §8f rank 2): kernel csrc/pred_learn.cu (forward, masked-L1 loss and the full backward in one launch), checked
against the reference's recorded ``learn`` call (tools/check_pred_learn.py, tests/test_gpu_learner.py): losses 7e-8,
all 112 gradient tensors <= 1e-5 relative, post-step weights 1.5e-8.  ``pred_optimizer_{i}_opt.th`` holds the Adam
state in torch.optim.Adam's state_dict format (reference :262).
"""
import copy
import os

import numpy as np
import torch

from .. import _lib
from ..modules.flat import ParamStack


class _PredAdam:
    """torch.optim.Adam-compatible ``state_dict`` of one agent's (GAT + decoder) optimiser (reference :84-90,
    files ``pred_optimizer_{i}_opt.th`` :262): parameter ids run over the GAT tensors, then the decoder tensors."""

    def __init__(self, owner, index):
        self.owner, self.index = owner, index

    def _entries(self):
        o, out, pid = self.owner, [], 0
        for kind, stack in (("gat", o.stack), ("dec", o.dec_stack)):
            for (name, shape), off in zip(stack.spec, stack.offsets):
                n = 1
                for d in shape:
                    n *= d
                out.append((pid, kind, shape, off, n))
                pid += 1
        return out

    def state_dict(self):
        o = self.owner
        o._learn_state()
        w, st = o._learn, {}
        for pid, kind, shape, off, n in self._entries():
            if w["step"] == 0:
                continue
            st[pid] = {"step": torch.tensor(float(w["step"])),
                       "exp_avg": w["m_" + kind][self.index, off:off + n].view(shape).detach().cpu().clone(),
                       "exp_avg_sq": w["v_" + kind][self.index, off:off + n].view(shape).detach().cpu().clone()}
        group = {"lr": float(o.args.lr_predict), "betas": (0.9, 0.999), "eps": float(o.args.optim_eps),
                 "weight_decay": float(getattr(o.args, "weight_decay", 0)), "amsgrad": False, "maximize": False, "foreach": None,
                 "capturable": False, "differentiable": False, "fused": None, "params": [e[0] for e in self._entries()]}
        return {"state": st, "param_groups": [group]}

    def load_state_dict(self, sd):
        o = self.owner
        o._learn_state()
        w = o._learn
        for pid, kind, shape, off, n in self._entries():
            if pid in sd["state"]:
                s_ = sd["state"][pid]
                w["m_" + kind][self.index, off:off + n] = s_["exp_avg"].reshape(-1).to(o.device)
                w["v_" + kind][self.index, off:off + n] = s_["exp_avg_sq"].reshape(-1).to(o.device)
                w["step"] = int(s_["step"])


class Prediction_policy:
    def __init__(self, args, logger=None):
        self.device = torch.device("cuda" if args.use_cuda else "cpu")
        if self.device.type != "cuda":
            raise RuntimeError("iplan_b200.Prediction_policy runs on CUDA only (no CPU path); set args.use_cuda=True")
        self.args = args
        self.logger = logger
        self.n_agents = args.n_agents
        self.max_vehicle_num = args.max_vehicle_num
        self.obs_shape = args.obs_shape_single
        if not getattr(args, "GAT_use_behavior", True):
            raise NotImplementedError("only the full iPLAN setting (GAT_use_behavior=True) is built")
        assert args.GAT_hidden_dim == 32 and args.attention_dim == 32, "kernel K1 is built for H = D = 32"
        self.GAT_input_dim = args.obs_shape_single + args.latent_dim          # reference :53-56
        self.stack = ParamStack("gat", self.n_agents, (self.GAT_input_dim,), device=self.device)
        self.pred_GAT = self.stack.nets
        self.tau = 0.01                                                       # nova/GAT_Net.py:93
        self.seed = int(getattr(args, "seed", 112358))
        self.calls = 0              # Philox counter: a fresh noise stream per call
        self.debug_gumbel = None    # [A,B,N,N-1,2] explicit gumbel noise for the next call (parity tests)
        self.capture_hard = False   # keep the hard-attention weights of the last call in .last_hard
        self.last_hard = None
        self._scratch = None      # kernel-to-kernel hand-off buffer of K1 (iplan_gat_scratch_floats)
        # ---- auxiliary trajectory-prediction learner (reference :63-90): decoder nets, one Adam over GAT + decoder
        self.dec_stack = ParamStack("pdec", self.n_agents, (args.obs_shape_single,), device=self.device)
        self.pred_decoder = self.dec_stack.nets
        self.prediction_batch_size = args.pred_batch_size
        self.pred_length = args.pred_length
        self._learn = None          # lazily allocated optimiser state / work buffers of learn()
        self.log_prefix = getattr(args, "log_prefix", "")
        self.log_stats_t = -getattr(args, "learner_log_interval", 0) - 1
        self.pred_optimizer = [_PredAdam(self, i) for i in range(self.n_agents)]
        self.debug_learn = None     # dict(select_idx=[A][P], gumbel=[A,P,N,N-1,2], keep=[A,P,pl,N,32] uint8) for parity runs
        self._stage = None        # device staging buffers of the pipelined numpy entry point

    # ---- device path: tensors laid out [A, B, N, *] (any strides) ------------------
    def gat_step(self, hist, beh_prev, h_prev, out, gumbel=None, dbg_hard=None, events=None):
        """out[a,b,n,:] = GAT_a(hist[a,b], beh_prev[a,b], h_prev[a,b]); all CUDA fp32.
        ``events``: optional three recorded ``torch.cuda.Event(enable_timing=True)``; they are re-recorded on the
        launching stream before the recurrence kernel, between the two kernels and after the attention kernel."""
        A, B, N, o = hist.shape
        if gumbel is not None:
            assert gumbel.is_contiguous() and tuple(gumbel.shape) == (A, B, N, N - 1, 2), gumbel.shape
        need = _lib.lib.iplan_gat_scratch_floats(B, A, N)
        if self._scratch is None or self._scratch.numel() < need or self._scratch.device != hist.device:
            self._scratch = torch.empty(need, device=hist.device, dtype=torch.float32)
        ev = [None, None, None] if events is None else [e.cuda_event for e in events]
        rc = _lib.lib.iplan_gat_step_ex(
            _lib.ptr(self.stack.flat), self.stack.stride(),
            _lib.view(hist), _lib.view(beh_prev), _lib.view(h_prev), _lib.view(out),
            _lib.ptr(gumbel), self.seed, self.calls, self.tau, _lib.ptr(dbg_hard),
            _lib.ptr(self._scratch), self._scratch.numel(),
            B, A, N, o, beh_prev.shape[-1], ev[0], ev[1], ev[2], _lib.stream())
        _lib.check(rc, "gat_step")
        self.calls += 1
        return out

    # ---- reference-compatible numpy entry point (reference :92-118) -----------------
    def GAT_latent_update(self, history_single, encoder_hidden, behavior_latent=None):
        dev = self.device
        gum = self.debug_gumbel
        self.debug_gumbel = None
        perm = (1, 0, 2, 3)       # [B,A,N,*] -> [A,B,N,*] views, no copy
        ins = (history_single, encoder_hidden, behavior_latent)
        # arrays this package returned last step (attention / behaviour latents) are still on the device: no upload
        on_dev = [_lib.device_shadow(x) for x in ins]
        host = [None if d is not None else _lib.as_host(x) for x, d in zip(ins, on_dev)]
        B = int(ins[0].shape[0])
        if gum is None and not self.capture_hard and B >= _lib.PIPELINE_MIN_ROWS:
            # one native call (csrc/host_api.cu): copy-in, K1 and copy-out overlap piece by piece over the envs
            A, N, o = int(ins[0].shape[1]), int(ins[0].shape[2]), int(ins[0].shape[3])
            D, L = int(ins[1].shape[-1]), int(ins[2].shape[-1])
            key = (B, A, N, o, D, L)
            if self._stage is None or self._stage[0] != key:
                self._stage = (key, [torch.empty(B, A, N, d, device=dev) for d in (o, D, L)])
            host = [None if h is None else h.contiguous() for h in host]
            full = []
            for d, st, h in zip(on_dev, self._stage[1], host):
                if d is not None:
                    _lib.io_bytes["h2d_saved"] += d.numel() * d.element_size()
                    full.append(d if d.dtype == torch.float32 and d.is_contiguous() else d.to(torch.float32).contiguous())
                else:
                    _lib.io_bytes["h2d"] += h.numel() * 4
                    full.append(st)
            out = torch.empty(B, A, N, D, device=dev)          # fresh: it becomes the shadow of the returned array
            out_h = torch.empty(B, A, N, D, dtype=torch.float32, pin_memory=True)
            need = _lib.lib.iplan_gat_scratch_floats(B, A, N)
            if self._scratch is None or self._scratch.numel() < need or self._scratch.device != out.device:
                self._scratch = torch.empty(need, device=dev, dtype=torch.float32)
            ends = _lib.wave_chunks(B, lambda e: (2 * e * A + 3) // 4)    # K1 recurrence: 2 CTAs per (env, agent-net), 4 resident per SM
            n_chunks = len(ends)
            _lib.check(_lib.lib.iplan_gat_latent_update_host(
                _lib.ptr(self.stack.flat), self.stack.stride(),
                _lib.host_ptr(host[0]), _lib.ptr(full[0]), _lib.host_ptr(host[1]), _lib.ptr(full[1]), _lib.host_ptr(host[2]), _lib.ptr(full[2]),
                _lib.ptr(out), _lib.host_ptr(out_h), self.seed, self.calls, self.tau, _lib.ptr(self._scratch), self._scratch.numel(),
                B, A, N, o, L, n_chunks, (_lib.C.c_int32 * n_chunks)(*ends), _lib.stream()), "gat_latent_update_host")
            self.calls += n_chunks
            _lib.io_bytes["d2h"] += out.numel() * 4
            return _lib.adopt_host(out_h, out)
        hs, eh, bl = (_lib.to_device(x) for x in ins)
        out = torch.empty_like(eh)
        dbg = None
        if self.capture_hard:
            B, A, N, _ = hs.shape
            dbg = torch.zeros(A, B, N, N - 1, device=dev)
            self.last_hard = dbg
        self.gat_step(hs.permute(perm), bl.permute(perm), eh.permute(perm), out.permute(perm), gum, dbg)
        return _lib.to_host(out, shadow=True)

    def _learn_state(self):
        """Optimiser state (Adam moments with the parameter buffers' layout) and work buffers of ``learn``."""
        if self._learn is None:
            dev, A = self.device, self.n_agents
            z = lambda t: torch.zeros_like(t)
            self._learn = dict(g_gat=z(self.stack.flat), g_dec=z(self.dec_stack.flat),
                               m_gat=z(self.stack.flat), v_gat=z(self.stack.flat), m_dec=z(self.dec_stack.flat), v_dec=z(self.dec_stack.flat),
                               ones_gat=torch.ones(self.stack.total, device=dev), ones_dec=torch.ones(self.dec_stack.total, device=dev),
                               sq=torch.zeros(A, device=dev), stats=torch.zeros(A, 8, device=dev), step=0, scratch=None)
        return self._learn

    def learn(self, batch, t_env):
        """Reference :168-253: per agent-net sample ``pred_batch_size`` (episode, time) transitions (:147), run the GAT
        and roll the decoder ``pred_length`` steps, masked L1 loss (:228-230), clip the GAT and the decoder gradients
        separately (:236-243), one Adam step over both (:84-90).  Returns the list of per-agent losses."""
        args, dev = self.args, self.device
        A, N, o, L, D = self.n_agents, self.max_vehicle_num, self.obs_shape, args.latent_dim, args.attention_dim
        P, pl = self.prediction_batch_size, self.pred_length
        hist = batch["history"][:, :-1]                       # [B, T, A, N, o]
        att = batch["attention_latent"][:, :-1]
        beh = batch["behavior_latent"][:, :-1]
        flag = batch["terminated"][:, :-1, :, 0].to(torch.float32)   # the reference multiplies the error by this flag (:196, :163)
        B, T = hist.shape[0], hist.shape[1]
        avail_len = T - pl - 1
        dbg = self.debug_learn or {}
        idx_rows = []
        for i in range(A):
            if "select_idx" in dbg:
                idx_rows.append(torch.as_tensor(dbg["select_idx"][i]).to(torch.int64))
            else:
                idx_rows.append(torch.as_tensor(np.random.choice(B * avail_len, size=P, replace=False)))   # :147
                for _ in range(pl):
                    np.random.random()                       # the decoder's teacher-forcing draws (prediction_net.py:55)
        sel = torch.stack(idx_rows).to(dev)                   # [A, P]
        b_i, t_i = torch.div(sel, avail_len, rounding_mode="floor"), sel % avail_len
        a_i = torch.arange(A, device=dev).view(A, 1).expand(A, P)
        x0 = hist[b_i, t_i, a_i].contiguous()                 # [A, P, N, o]
        att0 = att[b_i, t_i, a_i].contiguous()
        lat0 = beh[b_i, t_i, a_i].contiguous()
        target = torch.stack([hist[b_i, t_i + 1 + k, a_i] for k in range(pl)], dim=3).contiguous()    # [A, P, N, pl, o]
        mask = flag[b_i, t_i, a_i].contiguous()               # [A, P]
        scale = (o * pl) / (mask.sum(dim=1) * (N * pl * o) + 1e-10)
        w = self._learn_state()
        need = _lib.lib.iplan_pred_learn_scratch_floats(A, P, N, o, pl)
        if w["scratch"] is None or w["scratch"].numel() < need:
            w["scratch"] = torch.empty(need, device=dev)
        w["g_gat"].zero_(); w["g_dec"].zero_(); w["stats"].zero_()
        loss_sum = torch.zeros(A, device=dev)
        gum = dbg.get("gumbel")
        keep = dbg.get("keep")
        if gum is not None:
            gum = gum.to(dev, torch.float32).contiguous()
            assert tuple(gum.shape) == (A, P, N, N - 1, 2)
        if keep is not None:
            keep = keep.to(dev, torch.uint8).contiguous()
            assert tuple(keep.shape) == (A, P, pl, N, D)
        lib, st, ptr = _lib.lib, _lib.stream(), _lib.ptr
        _lib.check(lib.iplan_pred_learn(
            ptr(self.stack.flat), self.stack.stride(), ptr(self.dec_stack.flat), self.dec_stack.stride(),
            ptr(w["g_gat"]), ptr(w["g_dec"]), ptr(x0), ptr(lat0), ptr(att0), ptr(target), ptr(mask),
            ptr(gum), ptr(keep), ptr(scale.contiguous()), ptr(loss_sum), ptr(w["scratch"]), w["scratch"].numel(),
            self.seed, self.calls, self.tau, float(args.decoder_dropout), A, P, N, o, L, pl, st), "pred_learn")
        self.calls += 1
        self.last_grads = dict(gat=w["g_gat"].clone(), dec=w["g_dec"].clone())       # raw (unclipped) gradients, for parity checks
        w["step"] += 1
        for stack, g, m, v, ones, col in ((self.stack, w["g_gat"], w["m_gat"], w["v_gat"], w["ones_gat"], 0),
                                          (self.dec_stack, w["g_dec"], w["m_dec"], w["v_dec"], w["ones_dec"], 1)):
            _lib.check(lib.iplan_learner_adam(ptr(stack.flat), ptr(g), ptr(m), ptr(v), ptr(ones), ptr(w["sq"]), stack.stride(),
                                              stack.total, A, float(args.lr_predict), 0.9, 0.999, float(args.optim_eps), w["step"],
                                              float(args.max_grad_norm), 1.0, ptr(w["stats"]), col, st), "adam")
        losses = (loss_sum * scale).cpu()
        norms = w["stats"].cpu()
        out = [np.asarray(float(losses[i]), dtype=np.float32) for i in range(A)]
        self.train_info = dict(prediction_loss=float(losses.sum()), pred_encoder_grad_norm=float(norms[:, 0].sum()),
                               pred_decoder_grad_norm=float(norms[:, 1].sum()))
        if self.logger is not None and t_env - self.log_stats_t >= getattr(args, "learner_log_interval", 0):
            for k, v in self.train_info.items():
                self.logger.log_stat(self.log_prefix + k, v, t_env)
        return out

    # ---- checkpoints (reference :256-285) ----------------------------------------
    def save_models(self, path):
        for i, net in enumerate(self.pred_GAT):
            torch.save({k: v.detach().cpu() for k, v in net.state_dict().items()}, f"{path}/pred_GAT_{i}.th")
        for i, net in enumerate(self.pred_decoder):
            torch.save({k: v.detach().cpu() for k, v in net.state_dict().items()}, f"{path}/pred_decoder_{i}.th")
        for i in range(self.n_agents):
            torch.save(self.pred_optimizer[i].state_dict(), "{}/pred_optimizer_{}_opt.th".format(path, i))

    def load_models(self, paths, load_optimisers=False):
        if len(paths) == 1:
            paths = [copy.copy(paths[0]) for _ in range(self.n_agents)]
        for i, net in enumerate(self.pred_GAT):
            net.load_state_dict(torch.load(os.path.join(paths[i], f"pred_GAT_{i}.th"),
                                           map_location="cpu", weights_only=False))
        for i, net in enumerate(self.pred_decoder):
            f = os.path.join(paths[i], f"pred_decoder_{i}.th")
            if os.path.exists(f):
                net.load_state_dict(torch.load(f, map_location="cpu", weights_only=False))
        if load_optimisers:
            for i in range(self.n_agents):
                self.pred_optimizer[i].load_state_dict(torch.load("{}/pred_optimizer_{}_opt.th".format(paths[i], i),
                                                                  map_location="cpu", weights_only=False))
