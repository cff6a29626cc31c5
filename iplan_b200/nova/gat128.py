"""GAT_Net.forward at GAT_hidden_dim = attention_dim = 128 — BASELINE.json configs[4], the synthetic GAT + GRU
microbench (8192 envs x 32 agent-nets x 16 slots x 128-d features).  The op is the reference's
``GAT_Net.forward`` (nova/GAT_Net.py:41-142) with ``input_shape = GAT_hidden_dim = attention_dim = 128``
and ``max_vehicle_num = 16``; an "item" is one (env, agent-net) pair = 16 slots.

Split of the work (csrc/gat128.cu has the reasons):
  * the row x weight products over all slots — encode (:50), the factored input projections of the hard-attention GRU
    (W_ih [enc_i ; enc_j] = P_i + Q_j), q | k | v (:99-103), the GRUCell projections (:140) — are plain GEMMs and run
    through the library (cuBLAS fp32 via ``torch.bmm`` / ``torch.baddbmm``, TF32 off);
  * the bidirectional 15-step recurrence (:57-97), 80 % of the FLOPs, is ``iplan_gat128_recur`` (wgmma with W_hh
    resident in shared memory); attention and the GRUCell gates are ``iplan_gat128_attend`` / ``iplan_gat128_gates``.

Parameters use the reference's state_dict key names per agent-net (``load_state_dict(i, sd)`` accepts a reference
``GAT_Net(128, args)`` checkpoint).
"""
import math

import torch

from .. import _lib

H = 128
N = 16
K_RZ = -1.4426950408889634       # gate-activation scales folded into the projections (csrc/gat_common.cuh)
K_N = 2.8853900817779268


class GAT128:
    def __init__(self, n_agents, device="cuda", seed=0):
        if not str(device).startswith("cuda"):
            raise RuntimeError("iplan_b200.GAT128 runs on CUDA only (no CPU path)")
        self.A, self.device = n_agents, torch.device(device)
        g = torch.Generator().manual_seed(seed)
        A = n_agents

        def u(*shape, fan):
            return ((torch.rand(*shape, generator=g) * 2 - 1) / math.sqrt(fan)).to(self.device)

        # torch defaults of the reference module (Linear: U(+-1/sqrt(fan_in)); GRU / GRUCell: U(+-1/sqrt(hidden)))
        self.p = {"encoding.weight": u(A, H, H, fan=H), "encoding.bias": u(A, H, fan=H),
                  "hard_encoding.weight": u(A, 2, 2 * H, fan=2 * H), "hard_encoding.bias": u(A, 2, fan=2 * H),
                  "q.weight": u(A, H, H, fan=H), "k.weight": u(A, H, H, fan=H), "v.weight": u(A, H, H, fan=H), "v.bias": u(A, H, fan=H),
                  "rnn.weight_ih": u(A, 3 * H, H, fan=H), "rnn.weight_hh": u(A, 3 * H, H, fan=H),
                  "rnn.bias_ih": u(A, 3 * H, fan=H), "rnn.bias_hh": u(A, 3 * H, fan=H)}
        for sfx in ("", "_reverse"):
            self.p["hard_bi_GRU.weight_ih_l0" + sfx] = u(A, 3 * H, 2 * H, fan=H)
            self.p["hard_bi_GRU.weight_hh_l0" + sfx] = u(A, 3 * H, H, fan=H)
            self.p["hard_bi_GRU.bias_ih_l0" + sfx] = u(A, 3 * H, fan=H)
            self.p["hard_bi_GRU.bias_hh_l0" + sfx] = u(A, 3 * H, fan=H)
        self.tau = 0.01
        self.seed, self.calls = 112358 + seed, 0
        self._derived = None
        self._buf = None

    # ---- parameters ------------------------------------------------------------------------------------
    def state_dict(self, i):
        return {k: v[i].detach().cpu().clone() for k, v in self.p.items()}

    def load_state_dict(self, i, sd):
        for k, v in sd.items():
            self.p[k][i].copy_(torch.as_tensor(v))
        self._derived = None

    def _prepare(self):
        """Operand forms of the weights: gate scales folded into the hard-attention GRU's input projections and biases."""
        if self._derived is not None:
            return self._derived
        p, dev = self.p, self.device
        ks = torch.cat([torch.full((2 * H,), K_RZ), torch.full((H,), K_N)]).to(dev)            # per gate row
        d = {"WP": [], "WQ": [], "bQ": []}
        for sfx in ("", "_reverse"):
            wih, bih, bhh = p["hard_bi_GRU.weight_ih_l0" + sfx], p["hard_bi_GRU.bias_ih_l0" + sfx], p["hard_bi_GRU.bias_hh_l0" + sfx]
            d["WP"].append((wih[:, :, :H] * ks[None, :, None]).contiguous())                   # ego columns   (-> P)
            d["WQ"].append((wih[:, :, H:] * ks[None, :, None]).contiguous())                   # neighbour columns (-> Q)
            b = bih.clone()
            b[:, :2 * H] += bhh[:, :2 * H]                                                     # r | z: b_ih + b_hh; n: b_ih (b_hn stays inside r * (.))
            d["bQ"].append((b * ks[None, :]).contiguous())
        d["whh"] = torch.stack([p["hard_bi_GRU.weight_hh_l0"], p["hard_bi_GRU.weight_hh_l0_reverse"]], dim=1).contiguous()   # [A,2,384,128]
        d["bhn"] = torch.stack([p["hard_bi_GRU.bias_hh_l0"][:, 2 * H:], p["hard_bi_GRU.bias_hh_l0_reverse"][:, 2 * H:]], dim=1).contiguous()
        he = p["hard_encoding.weight"]                                                          # [A,2,256]: columns [fwd | rev]
        d["lw"] = torch.stack([he[:, 1, :H] - he[:, 0, :H], he[:, 1, H:] - he[:, 0, H:]], dim=1).contiguous()       # [A,2,128]
        d["Wqkv"] = torch.cat([p["q.weight"], p["k.weight"], p["v.weight"]], dim=1).contiguous()                    # [A,384,128]
        self._derived = d
        return d

    def _buffers(self, items):
        if self._buf is None or self._buf["items"] != items:
            A, M, dev = self.A, items * N, self.device
            z = lambda *s: torch.empty(*s, device=dev)
            self._buf = dict(items=items, enc=z(A, M, H), PQ=z(2, 2, A, M, 3 * H), dl=z(A, items, 2, N - 1, N),
                             qkv=z(A, M, 3 * H), xatt=z(A, M, H), gi=z(A, M, 3 * H), gh=z(A, M, 3 * H))
        return self._buf

    # ---- forward ---------------------------------------------------------------------------------------
    def forward(self, x, h_prev, gumbel=None, out=None, events=None):
        """x, h_prev [A, items, 16, 128] fp32 CUDA -> new hidden [A, items, 16, 128].
        ``gumbel`` None (in-kernel Philox) or [A, items, 16, 15, 2] explicit noise (reference draw order).
        ``events``: optional (e0, e1) CUDA events recorded around the recurrence kernel."""
        A, items = x.shape[0], x.shape[1]
        assert x.shape == (A, items, N, H) and h_prev.shape == x.shape and x.is_cuda and x.dtype == torch.float32
        assert x.is_contiguous() and h_prev.is_contiguous()
        prev_tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False                                          # the library GEMMs stay fp32
        try:
            d, w, p = self._prepare(), self._buffers(items), self.p
            M = items * N
            X, Hp = x.view(A, M, H), h_prev.view(A, M, H)
            torch.baddbmm(p["encoding.bias"][:, None, :], X, p["encoding.weight"].transpose(1, 2), out=w["enc"])
            w["enc"].relu_()                                                                    # :50
            for dr in range(2):
                torch.bmm(w["enc"], d["WP"][dr].transpose(1, 2), out=w["PQ"][0, dr])            # P  [A, M, 384]
                torch.baddbmm(d["bQ"][dr][:, None, :], w["enc"], d["WQ"][dr].transpose(1, 2), out=w["PQ"][1, dr])   # Q
            lib, st, P = _lib.lib, _lib.stream(), _lib.ptr
            if events is not None:
                events[0].record()
            _lib.check(lib.iplan_gat128_recur(P(w["PQ"][0]), P(w["PQ"][1]), P(d["whh"]), P(d["bhn"]), P(d["lw"]), P(w["dl"]),
                                              A, items, st), "gat128_recur")
            if events is not None:
                events[1].record()
            torch.bmm(w["enc"], d["Wqkv"].transpose(1, 2), out=w["qkv"])
            if gumbel is not None:
                assert gumbel.is_contiguous() and tuple(gumbel.shape) == (A, items, N, N - 1, 2)
            _lib.check(lib.iplan_gat128_attend(P(w["qkv"]), P(p["v.bias"]), P(w["dl"]), P(p["hard_encoding.bias"]), P(gumbel),
                                               self.seed, self.calls, self.tau, P(w["xatt"]), A, items, st), "gat128_attend")
            self.calls += 1
            torch.baddbmm(p["rnn.bias_ih"][:, None, :], w["xatt"], p["rnn.weight_ih"].transpose(1, 2), out=w["gi"])
            torch.baddbmm(p["rnn.bias_hh"][:, None, :], Hp, p["rnn.weight_hh"].transpose(1, 2), out=w["gh"])
            if out is None:
                out = torch.empty_like(x)
            _lib.check(lib.iplan_gat128_gates(P(w["gi"]), P(w["gh"]), P(h_prev), P(out), A * M, st), "gat128_gates")
            return out
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev_tf32

    @staticmethod
    def algorithmic(A, items):
        """(FLOPs of the recurrence kernel, FLOPs of the whole op, algorithmic HBM bytes of the whole op) per forward."""
        rows = A * items * N
        recur = rows * 2 * (N - 1) * 2 * 3 * H * H
        rest = rows * (2 * H * H + 2 * 2 * 2 * 3 * H * H + 3 * 2 * H * H + 2 * 2 * 3 * H * H + (N - 1) * 2 * H * 2)
        return recur, recur + rest, rows * 3 * H * 4
