"""pymarl ``EpisodeBatch`` with the reference's interface
(/root/reference/components/episode_buffer.py:6-205) over a device layout the kernels
read without re-packing.

Interface kept: ``EpisodeBatch(scheme, groups, batch_size, max_seq_length, data=None,
preprocess=None, device=...)``, ``update(data, bs, ts, mark_filled)``, ``batch[key]``,
``batch[(keys...)]``, ``batch[bs_slice, ts_slice]``, ``max_t_filled()``, ``to()``,
attributes ``scheme / groups / batch_size / max_seq_length / device / data``.

Layout: when the scheme carries the iPLAN feature keys
``history``, ``attention_latent`` and ``behavior_latent`` the three are views of ONE packed
tensor ``packed[A, B, T+1, Fp]`` whose rows are exactly the controller's input vector
(controllers/dcntrl_controller.py:187-213): per slot ``[history | attention | behaviour]``,
then the last-action one-hot, then the agent-id one-hot, zero padding to ``Fp``.
K1/K1b write their outputs into it, K1c and the learner GEMMs read rows from it; the
reference-shaped ``[B, T+1, A, N, *]`` tensors returned by ``batch["history"]`` etc. are
strided views of the same memory.
"""
from types import SimpleNamespace as SN

import numpy as np
import torch as th

PACKED_KEYS = ("history", "attention_latent", "behavior_latent")


def packed_row_stride(n_slots, slot_dim, n_actions, n_agents):
    f = n_slots * slot_dim + n_actions + n_agents
    return (f + 31) // 32 * 32


class EpisodeBatch:
    def __init__(self, scheme, groups, batch_size, max_seq_length, data=None, preprocess=None, device="cpu"):
        self.scheme = scheme.copy()
        self.groups = groups
        self.batch_size = batch_size
        self.max_seq_length = max_seq_length
        self.preprocess = {} if preprocess is None else preprocess
        self.device = device
        self._on_cuda = str(device).startswith("cuda")
        self.packed = None
        if data is not None:
            self.data = data
            return
        self.data = SN(transition_data={}, episode_data={})
        self._setup_data()

    # -------------------------------------------------------------------------------
    def _setup_data(self):
        scheme, groups = self.scheme, self.groups
        for k, (new_k, transforms) in self.preprocess.items():           # reference :32-49
            assert k in scheme
            vshape, dtype = scheme[k]["vshape"], scheme[k].get("dtype", th.float32)
            for tr in transforms:
                vshape, dtype = tr.infer_output_info(vshape, dtype)
            scheme[new_k] = {"vshape": vshape, "dtype": dtype}
            for extra in ("group", "episode_const"):
                if extra in scheme[k]:
                    scheme[new_k][extra] = scheme[k][extra]
        assert "filled" not in scheme, '"filled" is a reserved key for masking.'
        scheme["filled"] = {"vshape": (1,), "dtype": th.long}

        B, T1 = self.batch_size, self.max_seq_length
        pack = all(k in scheme for k in PACKED_KEYS) and "actions_onehot" in scheme and \
            str(self.device).startswith("cuda")
        if pack:
            A = groups[scheme["history"]["group"]]
            N, o = scheme["history"]["vshape"]
            D = scheme["attention_latent"]["vshape"][1]
            L = scheme["behavior_latent"]["vshape"][1]
            nact = scheme["actions_onehot"]["vshape"][0]
            S = o + D + L
            Fp = packed_row_stride(N, S, nact, A)
            self.packed = th.zeros(A, B, T1, Fp, dtype=th.float32, device=self.device)
            self.packed_dims = SN(A=A, N=N, o=o, D=D, L=L, S=S, n_actions=nact, F=N * S + nact + A, Fp=Fp,
                                  col_act=N * S, col_id=N * S + nact)
            ident = th.eye(A, device=self.device).view(A, 1, 1, A)
            self.packed[..., N * S + nact:N * S + nact + A] = ident          # agent-id one-hot (:211)
            slots = self.packed[..., :N * S].view(A, B, T1, N, S).permute(1, 2, 0, 3, 4)   # [B,T1,A,N,S]
            self.data.transition_data["history"] = slots[..., :o]
            self.data.transition_data["attention_latent"] = slots[..., o:o + D]
            self.data.transition_data["behavior_latent"] = slots[..., o + D:]
        for key, info in scheme.items():
            if pack and key in PACKED_KEYS:
                continue
            assert "vshape" in info, "Scheme must define vshape for {}".format(key)
            vshape = info["vshape"]
            if isinstance(vshape, int):
                vshape = (vshape,)
            group = info.get("group", None)
            if group:
                assert group in groups, "Group {} must have its number of members defined in _groups_".format(group)
                shape = (groups[group], *vshape)
            else:
                shape = tuple(vshape)
            dtype = info.get("dtype", th.float32)
            if info.get("episode_const", False):
                self.data.episode_data[key] = th.zeros((B, *shape), dtype=dtype, device=self.device)
            else:
                self.data.transition_data[key] = th.zeros((B, T1, *shape), dtype=dtype, device=self.device)

    def to(self, device):
        if self.packed is not None:
            raise RuntimeError("a packed EpisodeBatch lives on its CUDA device")
        for store in (self.data.transition_data, self.data.episode_data):
            for k, v in store.items():
                store[k] = v.to(device)
        self.device = device
        self._on_cuda = str(device).startswith("cuda")

    # -------------------------------------------------------------------------------
    def update(self, data, bs=slice(None), ts=slice(None), mark_filled=True):
        """Same contract as the reference's update (:87-112): values are converted to the
        scheme dtype on the batch's device and written with ``view_as`` semantics."""
        slices = self._parse_slices((bs, ts))
        basic = all(isinstance(x, slice) for x in slices)
        if self._on_cuda:
            from .. import _lib
        for k, v in data.items():
            if k in self.data.transition_data:
                target = self.data.transition_data
                if mark_filled:
                    target["filled"][tuple(slices)] = 1
                    mark_filled = False
                _slices = tuple(slices)
            elif k in self.data.episode_data:
                target = self.data.episode_data
                _slices = slices[0]
            else:
                raise KeyError("{} not found in transition or episode data".format(k))
            dtype = self.scheme[k].get("dtype", th.float32)
            if self._on_cuda:
                v = _lib.to_device(v, dtype=dtype, device=self.device)      # counts PCIe bytes
            elif th.is_tensor(v):
                v = v.to(device=self.device, dtype=dtype)
            else:
                v = th.as_tensor(np.asarray(v)).to(device=self.device, dtype=dtype)
            dest = target[k][_slices]
            self._check_safe_view(v, dest)
            if basic:
                dest.copy_(v.reshape(dest.shape))          # basic indexing: `dest` is a view of the store
            else:
                target[k][_slices] = v.reshape(dest.shape)
            if k in self.preprocess:
                new_k = self.preprocess[k][0]
                w = dest if basic else target[k][_slices]
                for tr in self.preprocess[k][1]:
                    w = tr.transform(w)
                if basic:
                    nd = target[new_k][_slices]
                    nd.copy_(w.view_as(nd))
                else:
                    target[new_k][_slices] = w.view_as(target[new_k][_slices])
                if self.packed is not None and new_k == "actions_onehot":
                    self._store_last_action(w, slices)

    def _store_last_action(self, onehot, slices):
        """Keep the packed rows' last-action columns equal to what the learner's input
        builder produces (controllers/dcntrl_controller.py:105-108): row t+1 gets
        onehot(action_t); row 0 gets onehot(action_0) — the reference's t = 0 quirk.
        (The rollout reads row 0 before action 0 is stored, i.e. zeros, as :203-206.)"""
        d = self.packed_dims
        T1 = self.max_seq_length
        ts = slices[1]
        t_idx = range(*ts.indices(T1)) if isinstance(ts, slice) else list(ts)
        oh = onehot.reshape(-1, len(t_idx), d.A, d.n_actions).permute(2, 0, 1, 3)      # [A,b,t,n_act]
        bsel = slices[0]           # write THROUGH an index expression: a list / tensor `bs` would make `packed[:, bs]` a copy
        if not isinstance(bsel, slice):
            bsel = th.as_tensor(bsel, device=self.packed.device).long()
        c0, c1 = d.col_act, d.col_act + d.n_actions
        for i, t in enumerate(t_idx):
            if t + 1 < T1:
                self.packed[:, bsel, t + 1, c0:c1] = oh[:, :, i]
            if t == 0:
                self.packed[:, bsel, 0, c0:c1] = oh[:, :, i]

    @staticmethod
    def _check_safe_view(v, dest):
        idx = len(v.shape) - 1
        for s in dest.shape[::-1]:
            if idx < 0 or v.shape[idx] != s:
                if s != 1:
                    raise ValueError("Unsafe reshape of {} to {}".format(v.shape, dest.shape))
            else:
                idx -= 1

    # -------------------------------------------------------------------------------
    def __getitem__(self, item):
        if isinstance(item, str):
            if item in self.data.episode_data:
                return self.data.episode_data[item]
            if item in self.data.transition_data:
                return self.data.transition_data[item]
            raise ValueError(item)
        if isinstance(item, tuple) and all(isinstance(it, str) for it in item):
            new = SN(transition_data={}, episode_data={})
            for key in item:
                if key in self.data.transition_data:
                    new.transition_data[key] = self.data.transition_data[key]
                elif key in self.data.episode_data:
                    new.episode_data[key] = self.data.episode_data[key]
                else:
                    raise KeyError("Unrecognised key {}".format(key))
            sch = {key: self.scheme[key] for key in item}
            grp = {self.scheme[key]["group"]: self.groups[self.scheme[key]["group"]]
                   for key in item if "group" in self.scheme[key]}
            return EpisodeBatch(sch, grp, self.batch_size, self.max_seq_length, data=new, device=self.device)
        item = self._parse_slices(item)
        new = SN(transition_data={k: v[tuple(item)] for k, v in self.data.transition_data.items()},
                 episode_data={k: v[item[0]] for k, v in self.data.episode_data.items()})
        return EpisodeBatch(self.scheme, self.groups, self._n_items(item[0], self.batch_size),
                            self._n_items(item[1], self.max_seq_length), data=new, device=self.device)

    @staticmethod
    def _n_items(ix, max_size):
        if isinstance(ix, (list, np.ndarray)):
            return len(ix)
        r = ix.indices(max_size)
        return 1 + (r[1] - r[0] - 1) // r[2]

    @staticmethod
    def _parse_slices(items):
        if isinstance(items, (slice, int, list, np.ndarray)) or th.is_tensor(items):
            items = (items, slice(None))
        if isinstance(items[1], list):
            raise IndexError("Indexing across Time must be contiguous")
        return [slice(it, it + 1) if isinstance(it, int) else it for it in items]

    def max_t_filled(self):
        return th.sum(self.data.transition_data["filled"], 1).max(0)[0]

    def __repr__(self):
        return "EpisodeBatch. Batch Size:{} Max_seq_len:{} Keys:{} Groups:{}".format(
            self.batch_size, self.max_seq_length, self.scheme.keys(), self.groups.keys())


class ReplayBuffer(EpisodeBatch):
    """Only its scheme is used on this path (run_ippo.py:188, :194)."""

    def __init__(self, scheme, groups, buffer_size, max_seq_length, preprocess=None, device="cpu"):
        super().__init__(scheme, groups, buffer_size, max_seq_length, preprocess=preprocess, device=device)
        self.buffer_size = buffer_size
