"""Parameter containers: one flat fp32 buffer per network type, stacked over agents.

The reference keeps ``n_agents`` independent ``nn.Module`` objects per network
(no parameter sharing: controllers/dcntrl_controller.py:176-185,
nova/prediction_policy.py:63-90, nova/stable_behavior_policy.py:55-80) and loops
over them in Python.  The kernels here index one ``[A, total]`` buffer by agent, so
each agent's module is a tree of ``nn.Parameter`` *views* into that buffer whose
``state_dict()`` has exactly the reference's keys, shapes and order — reference
checkpoints (``agent_i.th``, ``critic_i.th``, ``pred_GAT_i.th``,
``behavior_encoder_i.th``) load into it and files saved from it load in the reference.
"""
import math

import torch
import torch.nn as nn

from .. import _lib

H = 32    # GAT_hidden_dim == attention_dim == encoder_rnn_dim (kernel constant IPLAN_HID)
R = 64    # rnn_hidden_dim == mlp_hidden_dim (kernel constant IPLAN_RNN)


def gat_spec(in_dim):
    """nova/GAT_Net.py:18-39 — state_dict order."""
    g = []
    g += [("encoding.weight", (H, in_dim)), ("encoding.bias", (H,))]
    for sfx in ("", "_reverse"):
        g += [(f"hard_bi_GRU.weight_ih_l0{sfx}", (3 * H, 2 * H)), (f"hard_bi_GRU.weight_hh_l0{sfx}", (3 * H, H)),
              (f"hard_bi_GRU.bias_ih_l0{sfx}", (3 * H,)), (f"hard_bi_GRU.bias_hh_l0{sfx}", (3 * H,))]
    g += [("hard_encoding.weight", (2, 2 * H)), ("hard_encoding.bias", (2,)),
          ("q.weight", (H, H)), ("k.weight", (H, H)), ("v.weight", (H, H)), ("v.bias", (H,)),
          ("rnn.weight_ih", (3 * H, H)), ("rnn.weight_hh", (3 * H, H)), ("rnn.bias_ih", (3 * H,)), ("rnn.bias_hh", (3 * H,))]
    return g


def beh_spec(obs_dim, latent_dim):
    """nova/behavior_net.py:12-15 (EncoderRNN) — state_dict order."""
    return [("linear.weight", (H, obs_dim)), ("linear.bias", (H,)),
            ("rnn.weight_ih_l0", (3 * H, H)), ("rnn.weight_hh_l0", (3 * H, H)),
            ("rnn.bias_ih_l0", (3 * H,)), ("rnn.bias_hh_l0", (3 * H,)),
            ("out.weight", (latent_dim, H)), ("out.bias", (latent_dim,))]


def pdec_spec(obs_dim):
    """Prediction_Decoder -> DecoderRNN (nova/prediction_net.py:7-16, :29-35): hidden = attention_dim = H."""
    return [("decoder.linear.weight", (H, obs_dim)), ("decoder.linear.bias", (H,)),
            ("decoder.rnn.weight_ih_l0", (3 * H, H)), ("decoder.rnn.weight_hh_l0", (3 * H, H)),
            ("decoder.rnn.bias_ih_l0", (3 * H,)), ("decoder.rnn.bias_hh_l0", (3 * H,)),
            ("decoder.out.weight", (obs_dim, H)), ("decoder.out.bias", (obs_dim,))]


def bdec_spec(obs_dim, latent_dim, hidden=64):
    """Behavior_Latent_Decoder -> DecoderRNN (nova/behavior_net.py:25-47, :50-55): input = obs + latent, hidden = decoder_rnn_dim."""
    return [("decoder.linear.weight", (hidden, obs_dim + latent_dim)), ("decoder.linear.bias", (hidden,)),
            ("decoder.rnn.weight_ih_l0", (3 * hidden, hidden)), ("decoder.rnn.weight_hh_l0", (3 * hidden, hidden)),
            ("decoder.rnn.bias_ih_l0", (3 * hidden,)), ("decoder.rnn.bias_hh_l0", (3 * hidden,)),
            ("decoder.out.weight", (obs_dim, hidden)), ("decoder.out.bias", (obs_dim,))]


def bfc_spec(in_dim, hidden, latent_dim):
    """Encoder_3FC (nova/behavior_FC_net.py:6-20): W*o -> hidden -> hidden -> latent, state_dict order."""
    return [("linear_1.weight", (hidden, in_dim)), ("linear_1.bias", (hidden,)),
            ("linear_2.weight", (hidden, hidden)), ("linear_2.bias", (hidden,)),
            ("out.weight", (latent_dim, hidden)), ("out.bias", (latent_dim,))]


def bfcdec_spec(in_dim, latent_dim, hidden):
    """LILI_Latent_Decoder -> Decoder_3FC (nova/behavior_FC_net.py:23-60): W*o + latent -> hidden -> hidden -> W*o."""
    return [("decoder.linear_1.weight", (hidden, in_dim + latent_dim)), ("decoder.linear_1.bias", (hidden,)),
            ("decoder.linear_2.weight", (hidden, hidden)), ("decoder.linear_2.bias", (hidden,)),
            ("decoder.out.weight", (in_dim, hidden)), ("decoder.out.bias", (in_dim,))]


def trunk_spec(feat_dim):
    """MLPBase + RNNLayer (utils/mappo_utils/mlp.py:17-22,44-48; rnn.py:13-22)."""
    return [("base.feature_norm.weight", (feat_dim,)), ("base.feature_norm.bias", (feat_dim,)),
            ("base.mlp.fc1.0.weight", (R, feat_dim)), ("base.mlp.fc1.0.bias", (R,)),
            ("base.mlp.fc1.2.weight", (R,)), ("base.mlp.fc1.2.bias", (R,)),
            ("base.mlp.fc_h.0.weight", (R, R)), ("base.mlp.fc_h.0.bias", (R,)),
            ("base.mlp.fc_h.2.weight", (R,)), ("base.mlp.fc_h.2.bias", (R,)),
            ("base.mlp.fc2.0.0.weight", (R, R)), ("base.mlp.fc2.0.0.bias", (R,)),
            ("base.mlp.fc2.0.2.weight", (R,)), ("base.mlp.fc2.0.2.bias", (R,)),
            ("rnn.rnn.weight_ih_l0", (3 * R, R)), ("rnn.rnn.weight_hh_l0", (3 * R, R)),
            ("rnn.rnn.bias_ih_l0", (3 * R,)), ("rnn.rnn.bias_hh_l0", (3 * R,)),
            ("rnn.norm.weight", (R,)), ("rnn.norm.bias", (R,))]


def actor_spec(feat_dim, n_actions):
    """modules/agents/ippo_actor.py:32-40."""
    return trunk_spec(feat_dim) + [("act.action_out.linear.weight", (n_actions, R)),
                                   ("act.action_out.linear.bias", (n_actions,))]


def critic_spec(feat_dim):
    """modules/critics/ippo_critic.py:32-43; PopArt tensors utils/mappo_utils/popart.py:21-27."""
    return trunk_spec(feat_dim) + [("v_out.weight", (1, R)), ("v_out.bias", (1,)),
                                   ("v_out.stddev", (1,)), ("v_out.mean", (1,)),
                                   ("v_out.mean_sq", (1,)), ("v_out.debiasing_term", ())]


FROZEN = ("v_out.stddev", "v_out.mean", "v_out.mean_sq", "v_out.debiasing_term")
DEAD = ("base.mlp.fc_h.",)       # cloned into fc2 then never called (mlp.py:20-27): grad stays None
# PopArt on CUDA (utils/mappo_utils/popart.py:21-27): ``nn.Parameter(...).to(device)`` returns plain tensors, so a
# reference run with use_cuda=True has NO v_out.* entries in critic.state_dict(), 20 (not 26) optimiser params and a
# value head frozen at its initial value.  The CPU reference (the oracle, the golden fixtures) registers and trains
# them.  ``args.popart_cuda_quirk = True`` reproduces the CUDA behaviour (frozen head, 20-key checkpoints); loading
# accepts either checkpoint format in both modes.
POPART_KEYS = ("v_out.weight", "v_out.bias") + FROZEN


class AgentNet(nn.Module):
    """One agent's network: a module tree whose leaves are views into the stack."""

    def __init__(self, stack, index):
        super().__init__()
        object.__setattr__(self, "_stack", stack)
        self._index = index
        self._attach()

    def _attach(self):
        stack = self._stack
        for name in list(self._modules):
            del self._modules[name]
        flat = stack.flat[self._index]
        for (name, shape), off in zip(stack.spec, stack.offsets):
            n = int(math.prod(shape)) if len(shape) else 1
            leaf = flat[off:off + n].view(shape)
            parts = name.split(".")
            mod = self
            for p in parts[:-1]:
                if p not in mod._modules:
                    mod.add_module(p, nn.Module())
                mod = mod._modules[p]
            mod.register_parameter(parts[-1], nn.Parameter(leaf, requires_grad=name not in FROZEN))

    @property
    def device(self):
        return self._stack.flat.device

    def forward(self, *a, **k):
        raise RuntimeError("AgentNet holds parameters only; the arithmetic runs in libiplan_b200.so")

    def load_state_dict(self, state_dict, strict=True, **kw):
        """As nn.Module.load_state_dict; a critic checkpoint written by a CUDA run of the reference has no ``v_out.*``
        keys (see POPART_KEYS): those tensors then keep their current (initial) values."""
        if strict and self._stack.kind == "critic":
            missing = [k for k in self.state_dict() if k not in state_dict]
            if missing and all(k in POPART_KEYS for k in missing) and not [k for k in state_dict if k not in self.state_dict()]:
                return super().load_state_dict(state_dict, strict=False, **kw)
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _apply(self, fn, recurse=True):       # .cuda()/.to(): move the whole stack, then re-view
        self._stack._move(fn)
        return self


class ParamStack:
    """[A, total] fp32 buffer + per-agent AgentNet views; `kind` in gat|beh|actor|critic|pdec|bdec|bfc|bfcdec."""

    def __init__(self, kind, n_agents, dims, device="cpu"):
        self.kind, self.n_agents, self.dims = kind, n_agents, tuple(dims)
        self.spec = {"gat": gat_spec, "beh": beh_spec, "actor": actor_spec, "critic": critic_spec, "pdec": pdec_spec,
                     "bdec": bdec_spec, "bfc": bfc_spec, "bfcdec": bfcdec_spec}[kind](*dims)
        self.total, self.offsets = _lib.layout(kind, *(dims[:2] if kind == "bdec" else dims))
        assert len(self.offsets) == len(self.spec)
        # initialise on the host (orthogonal init = QR: dozens of tiny launches on a GPU), then move
        self.flat = torch.zeros(n_agents, self.total, dtype=torch.float32)
        self.nets = [AgentNet(self, i) for i in range(n_agents)]
        self.reset_parameters()
        if str(device) != "cpu":
            self.to(device)

    # -- placement ----------------------------------------------------------------
    def _move(self, fn):
        new = fn(self.flat)
        if new is not self.flat:
            self.flat = new
            for n in self.nets:
                n._attach()

    def to(self, device):
        self._move(lambda t: t.to(device))
        return self

    def stride(self):
        return self.flat.stride(0)

    def named_offsets(self):
        return {name: (off, shape) for (name, shape), off in zip(self.spec, self.offsets)}

    def trainable_mask(self, frozen_extra=()):
        """1.0 where Adam may move a value (excludes padding, PopArt statistics and
        the dead fc_h tensors, which the reference's optimiser never touches)."""
        m = torch.zeros(self.total)
        for (name, shape), off in zip(self.spec, self.offsets):
            if name in FROZEN or name.startswith(DEAD[0]) or name in frozen_extra:
                continue
            n = int(math.prod(shape)) if len(shape) else 1
            m[off:off + n] = 1.0
        return m

    # -- initialisation as the reference does it -------------------------------------
    @torch.no_grad()
    def reset_parameters(self):
        for a in range(self.n_agents):
            sd = dict(self.nets[a].named_parameters())
            for name, p in sd.items():
                self._init_tensor(name, p)

    def _init_tensor(self, name, p):
        k = self.kind
        if k in ("gat", "beh", "pdec", "bdec", "bfc", "bfcdec"):
            # torch defaults: Linear U(+-1/sqrt(fan_in)); GRU/GRUCell U(+-1/sqrt(hidden))
            if "GRU" in name or name.startswith("rnn.") or ".rnn." in name:
                hidden = dict(self.spec)["decoder.rnn.weight_hh_l0"][1] if k in ("pdec", "bdec") else H
                bound = 1.0 / math.sqrt(hidden)
            else:
                fan_in = dict(self.spec)[name.rsplit(".", 1)[0] + ".weight"][1]
                bound = 1.0 / math.sqrt(fan_in)
            p.uniform_(-bound, bound)
            return
        if name in FROZEN:
            p.fill_(1.0 if name.endswith("stddev") else 0.0)
        elif name.endswith("norm.weight") or name.endswith(".2.weight"):
            p.fill_(1.0)                                            # LayerNorm
        elif "bias" in name:
            p.zero_()                                               # mlp.py:15, rnn.py:16, act/critic init_
        elif name.startswith("act."):
            nn.init.orthogonal_(p, gain=0.01)                       # config/algs/ippo.yaml:23 gain
        elif name.startswith("v_out."):
            nn.init.orthogonal_(p, gain=1.0)                        # ippo_critic.py:37-41
        elif name.startswith("rnn.rnn."):
            nn.init.orthogonal_(p)                                  # rnn.py:17-19
        else:
            nn.init.orthogonal_(p, gain=math.sqrt(2.0))             # mlp.py:12-16 (ReLU gain)
