"""Behavioural-incentive module, hard-update variant (the iPLAN-Hard ablation) — mirror of the reference's
``nova/behavior_policy.Behavior_policy`` (reference run_ippo.py:200-209 builds it when ``soft_update_enable`` is False).

Constructor, networks, optimiser state and checkpoint files are those of the soft-update class
(``stable_behavior_policy.Behavior_policy``, reference nova/behavior_policy.py:14-77).  What differs:

* ``latent_update`` (reference :78-116) returns the encoder's new soft-max latent and ignores ``prev_latent``.  It is the
  soft update with coefficient 1: kernel K1b computes ``0 * prev + z * 1``, which is ``z`` bit for bit for finite
  ``prev``, so the rollout needs no kernel of its own.
* ``learn`` (reference :119-215) cuts each episode into non-overlapping windows of W = max_history_len steps: the decoder
  reads window j with latent_j, the encoder then reads window j and gives latent_{j+1} (latent_0 = 0), the target is
  window j+1.  Same register-tiled kernels as the soft update (csrc/beh_learn_tile.cu, entry
  ``iplan_beh_learn_windows`` with the geometry (W, 0)); the arithmetic is specified by
  tools/beh_hard_oracle.py::behavior_learn_hard_agent.
"""
import torch

import numpy as np

from .stable_behavior_policy import Behavior_policy as _SoftBehaviorPolicy


class Behavior_policy(_SoftBehaviorPolicy):
    def __init__(self, args, logger=None):
        super().__init__(args, logger)
        self.soft_update_coef = 1.0          # the new latent replaces the previous one (rollout and learn)

    def learn(self, batch, t_env):
        """Reference :119-215, per agent-net with T = batch.max_seq_length - 1 and W = max_history_len:

        * the episode is T / W windows; T % W != 0 raises, as the reference's ``reshape`` does (:142), and so does
          T < 2 W (no window has a successor);
        * positions j = 0 .. T/W - 2 are trained, hidden states of encoder and decoder carried across them;
        * the mask is ``terminated`` on Highway and ``1 - terminated`` on MPE (:146-149), cut to its first
          (T/W - 1) W rows (:144), so the target at row t is weighted by the mask at row t - W;
        * loss = sum |next - pred| m / (N o sum m + 1e-10) o N (:184-186), one normalisation over all windows and no
          stability term;
        * encoder and decoder gradients clipped separately to max_grad_norm, then one Adam step (lr_behavior) over both.

        Returns ONE list of A float32 numpy scalars, as the reference does (:215).  The reference's runner unpacks three
        values from it (run_ippo.py:271), which only works when A == 3.  Logs behavior_loss, behavior_encoder_grad_norm
        and behavior_decoder_grad_norm."""
        args = self.args
        if float(getattr(args, "behavior_variation_penalty", 0)) != 0.0:
            raise NotImplementedError("only behavior_variation_penalty = 0 (the iPLAN setting) is built")
        A, N, o, W = self.n_agents, self.max_vehicle_num, args.obs_shape_single, self.max_history_len
        hist = batch["history"][:, :-1]                                  # [B, T, A, N, o]
        B, T = hist.shape[0], hist.shape[1]
        if T % W != 0:
            raise RuntimeError(f"Behavior_policy.learn (hard update): episode of {T} steps is not a whole number of "
                               f"windows of {W} steps")
        n_pos = T // W - 1
        if n_pos < 1:
            raise RuntimeError(f"Behavior_policy.learn (hard update): episode of {T} steps has fewer than two windows of {W} steps")
        term = batch["terminated"][:, :-1, :, 0].to(torch.float32)      # [B, T, A]
        mask = (1.0 - term) if args.env == "MPE" else term
        hist_a = hist.permute(2, 0, 1, 3, 4).contiguous()
        mask_a = mask.permute(2, 0, 1)                                   # [A, B, T]
        cut = n_pos * W
        lagged = torch.zeros_like(mask_a)                                # read at the target row t: mask[t - W]
        lagged[:, :, W:] = mask_a[:, :, :cut]
        msum = mask_a[:, :, :cut].sum(dim=(1, 2)) * (N * o)              # [A] elements the reference's mask keeps
        scale = ((o * N) / (msum + 1e-10)).unsqueeze(1).expand(A, n_pos).contiguous()
        bl, _, norms = self._learn_step(hist_a, lagged.contiguous(), scale, n_pos, windows=(W, 0))
        behavior_loss = [np.asarray(float(bl[i]), dtype=np.float32) for i in range(A)]
        self._log(t_env, dict(behavior_loss=float(bl.sum()), behavior_encoder_grad_norm=float(norms[:, 0].sum()),
                              behavior_decoder_grad_norm=float(norms[:, 1].sum())))
        return behavior_loss
