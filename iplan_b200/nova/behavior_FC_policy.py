"""Behavioural-incentive module, fully-connected variant (the iPLAN-FC ablation) — mirror of the reference's
``nova/behavior_FC_policy.Behavior_policy`` (reference run_ippo.py:200-203 builds it when ``behavior_fully_connected`` is
True, whatever ``soft_update_enable`` says).

Same constructor, optimiser state, checkpoint files and logging as the soft-update class
(``stable_behavior_policy.Behavior_policy``); the networks are the reference's two small MLPs (nova/behavior_FC_net.py):
``Encoder_3FC`` (W*o -> E -> E -> L: tanh, tanh, soft-max) and ``LILI_Latent_Decoder`` (W*o + L -> Dh -> Dh -> W*o: tanh,
tanh, linear), E = encoder_rnn_dim = 32 and Dh = decoder_rnn_dim = 64.  What differs from the GRU module:

* ``latent_update`` (reference :80-106) is the encoder on each window: no hidden state, no soft update.  ``prev_latent`` is
  ignored and ``encoder_hidden`` comes back unchanged.  Kernel ``iplan_behavior_fc_step`` (csrc/behavior_fc.cu).
* ``learn`` (reference :146-236) is one fused forward + backward (``iplan_beh_fc_learn``), then the soft module's clip and
  Adam step.  The arithmetic is specified by tools/beh_fc_oracle.py.
"""
import numpy as np
import torch

from .. import _lib
from ..modules.flat import ParamStack
from .stable_behavior_policy import Behavior_policy as _SoftBehaviorPolicy


class Behavior_policy(_SoftBehaviorPolicy):
    def _build_nets(self, args):
        if args.encoder_rnn_dim != 32 or args.decoder_rnn_dim != 64:
            raise ValueError(f"iPLAN-FC kernels are built for encoder_rnn_dim 32 and decoder_rnn_dim 64, not "
                             f"{args.encoder_rnn_dim} and {args.decoder_rnn_dim}")
        in_dim = args.obs_shape_single * args.max_history_len
        self.stack = ParamStack("bfc", self.n_agents, (in_dim, args.encoder_rnn_dim, args.latent_dim), device=self.device)
        self.dec_stack = ParamStack("bfcdec", self.n_agents, (in_dim, args.latent_dim, args.decoder_rnn_dim), device=self.device)

    def _learn_step(self, *a, **k):
        raise RuntimeError("the GRU behaviour learner (iplan_beh_learn) does not apply to the fully-connected module's "
                           "parameters; Behavior_policy.learn runs iplan_beh_fc_learn")

    # ---- device path: tensors laid out [A, B, N, *] ----------------------------------
    def behavior_step(self, window, hid_io, lat_prev, lat_out, win_stride_step=0, win_pad=0):
        """The soft module's signature, so that the device runner calls either: window [A,B,N,W*o] (or, with
        ``win_stride_step`` != 0, the [A,B,N,o] view of the oldest real row of a time-strided store, ``win_pad`` leading
        zero rows), lat_out [A,B,N,L].  ``hid_io`` and ``lat_prev`` are not read: the encoder has no state."""
        A, B, N, _ = window.shape
        rc = _lib.lib.iplan_behavior_fc_step(
            _lib.ptr(self.stack.flat), self.stack.stride(), _lib.view(window), int(win_stride_step), int(win_pad),
            _lib.view(lat_out), B, A, N, self.args.obs_shape_single, self.latent_dim, self.max_history_len,
            self.args.encoder_rnn_dim, _lib.stream())
        _lib.check(rc, "behavior_fc_step")
        return lat_out, hid_io

    # ---- reference-compatible entry point (reference :80-106) -------------------------
    def latent_update(self, history, encoder_hidden=None, prev_latent=None):
        """history [B,A,N,W,o] -> (read-only numpy latent [B,A,N,L] with a device shadow, encoder_hidden unchanged)."""
        hist = _lib.to_device(history).contiguous()
        B, A, N, W, o = hist.shape
        new = torch.empty(B, A, N, self.latent_dim, device=self.device)
        perm = (1, 0, 2, 3)
        self.behavior_step(hist.view(B, A, N, W * o).permute(perm), None, None, new.permute(perm))
        return _lib.to_host(new, shadow=True), encoder_hidden

    def learn(self, batch, t_env):
        """Reference :146-236, per agent-net with T = batch.max_seq_length - 1, W = max_history_len and
        n_pos = T - 1 - W positions (n_pos < 1 raises: the reference divides by zero there):

        * at position j the decoder reads the window ending at j and latent_{j-1} = encoder(window ending at j-1),
          latent_{-1} = 0, and predicts the window ending at j+1;
        * loss = mean over j of sum |next - pred| / (B N W o + 1e-10) o N.  ``terminated`` has no effect: the reference's
          mask loop writes the current-window mask twice (:135-140), so the next-window mask stays all ones;
        * encoder and decoder gradients clipped separately to max_grad_norm, then one Adam step (lr_behavior) over both.

        Returns (behavior_loss, [], total_loss): lists of A float32 numpy scalars and an empty stability list."""
        args, dev = self.args, self.device
        A, N, o, L, W = self.n_agents, self.max_vehicle_num, args.obs_shape_single, self.latent_dim, self.max_history_len
        hist = batch["history"][:, :-1]                                  # [B, T, A, N, o]
        B, T = hist.shape[0], hist.shape[1]
        n_pos = T - 1 - W
        if n_pos < 1:
            raise RuntimeError(f"Behavior_policy.learn (fully connected): episode of {T} steps has no position to train "
                               f"with windows of {W} steps (needs T - 1 - W >= 1)")
        hist_a = hist.permute(2, 0, 1, 3, 4).to(device=dev, dtype=torch.float32).contiguous()
        scale = float(o * N) / (float(B * N * W * o) + 1e-10) / n_pos
        w = self._learn_state()
        w["g_enc"].zero_(); w["g_dec"].zero_(); w["stats"].zero_()
        b_loss = torch.zeros(A, device=dev)
        ptr = _lib.ptr
        _lib.check(_lib.lib.iplan_beh_fc_learn(
            ptr(self.stack.flat), self.stack.stride(), ptr(self.dec_stack.flat), self.dec_stack.stride(), ptr(w["g_enc"]),
            ptr(w["g_dec"]), ptr(hist_a), scale, ptr(b_loss), A, B, T, N, o, L, W, args.encoder_rnn_dim,
            args.decoder_rnn_dim, _lib.stream()), "beh_fc_learn")
        self.learn_calls += 1
        self._adam_step()
        bl, norms = b_loss.cpu(), w["stats"].cpu()
        behavior_loss = [np.asarray(float(bl[i]), dtype=np.float32) for i in range(A)]
        total_loss = [np.asarray(float(bl[i]), dtype=np.float32) for i in range(A)]
        self._log(t_env, dict(behavior_loss=float(bl.sum()), stability_loss=0.0, behavior_total=float(bl.sum()),
                              behavior_encoder_grad_norm=float(norms[:, 0].sum()),
                              behavior_decoder_grad_norm=float(norms[:, 1].sum())))
        return behavior_loss, [], total_loss
