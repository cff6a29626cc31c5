"""ctypes binding of libiplan_b200.so (include/iplan_b200.h).

The CUDA library is the product: there is NO fallback.  If the shared object is
missing this module raises at import; if a call fails it raises RuntimeError with
the library's error text.  torch is used only for device memory and streams.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "build", "libiplan_b200.so")

if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(or `make -C iplan_b200/csrc`).  iplan_b200 has no CPU / PyTorch fallback.")

lib = C.CDLL(LIB_PATH)


class View(C.Structure):
    """iplan_view: element [agent][env][slot][0..dim) of a strided fp32 array."""
    _fields_ = [("ptr", C.c_void_p), ("stride_agent", C.c_int64),
                ("stride_env", C.c_int64), ("stride_slot", C.c_int64)]


_p, _i, _i64, _u64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.c_float

_SIGNATURES = {
    "iplan_abi_version": (C.c_int, []),
    "iplan_last_error": (C.c_char_p, []),
    "iplan_launch_count": (_i64, []),
    "iplan_gat_layout": (_i64, [_i, _p]),
    "iplan_beh_layout": (_i64, [_i, _i, _p]),
    "iplan_actor_layout": (_i64, [_i, _i, _p]),
    "iplan_critic_layout": (_i64, [_i, _p]),
    "iplan_gat_scratch_floats": (_i64, [_i, _i, _i]),
    "iplan_gat_step": (_i, [_p, _i64, View, View, View, View, _p, _u64, _u64, _f, _p, _p, _i64,
                            _i, _i, _i, _i, _i, _p]),
    "iplan_gat_step_ex": (_i, [_p, _i64, View, View, View, View, _p, _u64, _u64, _f, _p, _p, _i64,
                               _i, _i, _i, _i, _i, _p, _p, _p, _p]),
    "iplan_gat128_recur": (_i, [_p, _p, _p, _p, _p, _p, _i, _i64, _p]),
    "iplan_gat128_attend": (_i, [_p, _p, _p, _p, _p, _u64, _u64, _f, _p, _i, _i64, _p]),
    "iplan_gat128_gates": (_i, [_p, _p, _p, _p, _i64, _p]),
    "iplan_behavior_step": (_i, [_p, _i64, View, View, View, View, _f, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_behavior_step_ex": (_i, [_p, _i64, View, _i64, _i, View, View, View, _f, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_gat_latent_update_host": (_i, [_p, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _u64, _u64, _f, _p, _i64, _i, _i, _i, _i, _i, _i, _p, _p]),
    "iplan_behavior_latent_update_host": (_i, [_p, _i64, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_d2h_batch": (_i, [_p, _p, _p, _i, _p]),
    "iplan_controller_step": (_i, [_p, _i64, _p, _i64, _p, _i64, _i64, _p, _p, _p, _p, _i64, _i64, _i64, _i64,
                                   _p, _p, _u64, _u64, _i, _p, _p, _p, _p, _p, _p,
                                   _i, _i, _i, _i, _p]),
    "iplan_obs_history_step": (_i, [_p, _i, _i, _i, _i, _p, _p, _p, _p, _p, _i, _i, _p]),
    "iplan_pdec_layout": (_i64, [_i, _p]),
    "iplan_pred_learn_scratch_floats": (_i64, [_i, _i, _i, _i, _i]),
    "iplan_pred_learn": (_i, [_p, _i64, _p, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _u64, _u64, _f, _f,
                              _i, _i, _i, _i, _i, _i, _p]),
    "iplan_bdec_layout": (_i64, [_i, _i, _p]),
    "iplan_beh_learn_scratch_floats": (_i64, [_i, _i, _i, _i, _i, _i, _i]),
    "iplan_beh_learn_set_impl": (_i, [_i]),
    "iplan_beh_learn": (_i, [_p, _i64, _p, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _u64, _u64, _f, _f, _f,
                             _i, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_beh_learn_tile_scratch_floats": (_i64, [_i, _i, _i, _i, _i, _i, _i]),
    "iplan_beh_learn_windows": (_i, [_p, _i64, _p, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _u64, _u64, _f, _f, _f,
                                     _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_bfc_layout": (_i64, [_i, _i, _i, _p]),
    "iplan_bfcdec_layout": (_i64, [_i, _i, _i, _p]),
    "iplan_behavior_fc_step": (_i, [_p, _i64, View, _i64, _i, View, _i, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_beh_fc_learn": (_i, [_p, _i64, _p, _i64, _p, _p, _p, _f, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "iplan_learner_row_stats": (_i, [_p, _i64, _i, _i, _i64, _i, _p, _p]),
    "iplan_learner_x_split": (_i, [_p, _i64, _p, _p, _p]),
    "iplan_learner_fc1_forward": (_i, [_p, _i64, _p, _i64, _p, _p, _i64, _i, _i, _i64, _i, _p, _p, _p, _p, _p, _p, _p]),
    "iplan_learner_tail": (_i, [_p, _i, _p]),
    "iplan_learner_gather_rows": (_i, [_p, _p]),
    "iplan_learner_fc1_backward": (_i, [_p, _i64, _p, _i64, _p, _p, _p, _p, _i64, _i, _i, _i64, _i,
                                        _p, _p, _p, _p, _p, _p, _p]),
    "iplan_learner_gae": (_i, [_p, _p, _p, _f, _f, _i, _i, _i, _i, _p, _p, _p, _p]),
    "iplan_learner_adv_finalize": (_i, [_p, C.c_double, _p, _i, _p]),
    "iplan_learner_adam": (_i, [_p, _p, _p, _p, _p, _p, _i64, _i64, _i, _f, _f, _f, _f, _i, _f, _f, _p, _i, _p]),
}


class LearnerCtx(C.Structure):
    """iplan_learner_ctx (include/iplan_b200.h)."""
    _fields_ = [("actor", _p), ("critic", _p), ("actor_stride", _i64), ("critic_stride", _i64),
                ("g_actor", _p), ("g_critic", _p),
                ("feat_dim", _i), ("n_actions", _i), ("n_agents", _i), ("T1", _i), ("n_eps", _i), ("n_train_eps", _i),
                ("rnn_a", _p), ("rnn_c", _p), ("rnn_stride_agent", _i64), ("rnn_ld", _i),
                ("actions", _p), ("avail", _p),
                ("Z1", _p), ("A1", _p), ("Z2", _p), ("A2", _p), ("GI", _p), ("GH", _p),
                ("stat", _p), ("SM", _p),
                ("logp_out", _p), ("ent_out", _p), ("value_out", _p),
                ("old_logp", _p), ("old_value", _p), ("returns", _p), ("adv_raw", _p), ("alive", _p),
                ("norm", _p), ("stats", _p),
                ("clip", _f), ("ent_coef", _f), ("v_coef", _f), ("huber_delta", _f), ("grad_scale", _f),
                ("train_rows", _p)]


class GatherArgs(C.Structure):
    """iplan_gather_args (include/iplan_b200.h)."""
    _fields_ = [("idx", _p), ("rows_src", _i64), ("rows_dst", _i64), ("n_agents", _i), ("ldx", _i), ("n_actions", _i),
                ("Xh", _p), ("Xl", _p), ("Xh_out", _p), ("Xl_out", _p), ("stat", _p), ("stat_out", _p),
                ("rnn_a", _p), ("rnn_c", _p), ("rnn_a_out", _p), ("rnn_c_out", _p),
                ("actions", _p), ("actions_out", _p), ("avail", _p), ("avail_out", _p),
                ("scalars", _p * 5), ("scalars_out", _p * 5)]


def _bind(signatures):
    for name, (res, args) in signatures.items():
        fn = getattr(lib, name)         # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args


_bind(_SIGNATURES)

ABI_VERSION = lib.iplan_abi_version()


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError(f"iplan_b200 {what} failed (rc={rc}): {lib.iplan_last_error().decode()}")


def launch_count():
    return int(lib.iplan_launch_count())


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_cuda, "iplan_b200 kernels take CUDA tensors only"
    return C.c_void_p(t.data_ptr())


def view(t):
    """[A, B, N, dim] fp32 CUDA tensor (any strides, innermost contiguous) -> iplan_view."""
    assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 4, (t.shape, t.dtype, t.device)
    assert t.stride(3) == 1 or t.shape[3] == 1, "innermost dimension must be contiguous"
    return View(t.data_ptr(), t.stride(0), t.stride(1), t.stride(2))


io_bytes = {"h2d": 0, "d2h": 0, "h2d_saved": 0}      # host<->device traffic of the reference-facing (numpy) API

# ---- device shadows of arrays this package handed out ------------------------------------------
# The reference's runner passes several results straight back into the next call (attention_latent, behavior_latent,
# rnn states: runners/ippo_parallel_runner.py:222-266).  A numpy array returned by ``to_host(t, shadow=True)`` is made
# READ-ONLY and remembered together with the (immutable) device tensor it was copied from; when the same array object
# comes back, ``to_device`` returns that tensor instead of re-uploading it.  Identity + read-only means the content
# cannot have changed; a copy or a modified array is simply uploaded as before.
SHADOW = True
_shadow = {}


def _register_shadow(arr, dev_t):
    import weakref
    key = id(arr)
    arr.flags.writeable = False

    def _drop(_ref, key=key):
        _shadow.pop(key, None)
    _shadow[key] = (weakref.ref(arr, _drop), dev_t)


def device_shadow(x):
    """The device tensor an earlier ``to_host(..., shadow=True)`` produced `x` from, or None."""
    import numpy as np
    if not SHADOW or not isinstance(x, np.ndarray):
        return None
    e = _shadow.get(id(x))
    if e is not None and e[0]() is x and not x.flags.writeable:
        return e[1]
    return None


def to_device(x, dtype=torch.float32, device="cuda"):
    """numpy / CPU tensor -> CUDA tensor of `dtype`, counting the bytes that cross PCIe.

    The host buffer is reusable when this returns (the reference's ``th.tensor(x).to(device)`` semantics).  Every call of
    the numpy API returns with the compute stream drained, so the copy is simply issued on it."""
    import numpy as np
    sh = device_shadow(x)
    if sh is not None:                       # an array we returned, handed straight back: already on the device
        io_bytes["h2d_saved"] += sh.numel() * sh.element_size()
        return sh if sh.dtype == dtype else sh.to(dtype)
    if torch.is_tensor(x):
        if x.is_cuda:
            return x.to(dtype)
        t = x
    else:
        t = torch.as_tensor(np.asarray(x))
    if t.dtype != dtype:
        t = t.to(dtype)
    io_bytes["h2d"] += t.numel() * t.element_size()
    return t.to(device)


def to_host(t, shadow=False):
    """CUDA tensor -> fresh numpy array (page-locked, from torch's caching host allocator, so that
    the copy runs at PCIe speed and a later ``to_device`` of the same array does too).
    ``shadow=True``: `t` will not be written again by the caller; the returned array is read-only and ``to_device``
    of that same array object returns `t` without a copy (see ``device_shadow``)."""
    return to_host_many([t], shadows=(0,) if shadow else ())[0]


def adopt_host(h, dev_t):
    """Pinned CPU tensor `h` filled from the immutable device tensor `dev_t` -> read-only numpy array with a shadow."""
    arr = h.numpy()
    if SHADOW:
        _register_shadow(arr, dev_t)
    return arr


def pinned_numpy(t):
    """Copy of a (CUDA or CPU) tensor as a numpy array in page-locked host memory."""
    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    h.copy_(t)
    if t.is_cuda:
        torch.cuda.current_stream().synchronize()
    return h.numpy()


_device_index = None


def stream():
    """The current CUDA stream of this process's device as a raw handle.  (``torch.cuda.current_stream()`` costs ~13 us
    of interpreter time per call; this is the same lookup without the wrapper object.  One device per process.)"""
    global _device_index
    if _device_index is None:
        _device_index = torch.cuda.current_device()
    return C.c_void_p(torch._C._cuda_getCurrentRawStream(_device_index))


def host_ptr(t):
    """Address of a CPU tensor's storage (None -> NULL)."""
    if t is None:
        return None
    assert not t.is_cuda and t.is_contiguous() and t.dtype == torch.float32, (t.device, t.dtype)
    return C.c_void_p(t.data_ptr())


def to_host_many(tensors, shadows=()):
    """Several small CUDA tensors -> fresh page-locked numpy arrays with ONE stream synchronize
    (csrc/host_api.cu iplan_d2h_batch).  ``shadows``: indices whose arrays are registered as device shadows."""
    n = len(tensors)
    tensors = [t.contiguous() for t in tensors]
    hosts = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in tensors]
    dst = (C.c_void_p * n)(*[h.data_ptr() for h in hosts])
    src = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
    nb = (C.c_int64 * n)(*[t.numel() * t.element_size() for t in tensors])
    check(lib.iplan_d2h_batch(dst, src, nb, n, stream()), "d2h_batch")
    out = []
    for i, (h, t) in enumerate(zip(hosts, tensors)):
        io_bytes["d2h"] += t.numel() * t.element_size()
        arr = h.numpy()
        if i in shadows and SHADOW:
            _register_shadow(arr, t)
        out.append(arr)
    return out


# ---- chunk-pipelined host <-> device calls (the reference-facing numpy API) --------------------
PIPELINE_MIN_ROWS = 128      # below this many envs a call is one copy-in / launch / copy-out


MAX_PIPELINE_CHUNKS = 16     # csrc/host_api.cu MAX_CHUNKS
_sm_count = None


def wave_chunks(n_envs, ctas_of):
    """End indices of the env pieces of a pipelined call of K1; ``ctas_of(envs)`` = its grid size in units of one SM's resident CTAs.
    Consecutive launches on one stream do not overlap, so every piece pays for a whole last wave.  The pieces therefore hold
    whole waves (never more waves in total than a single launch), the LAST piece is what does not fill the other waves (its
    copy-out is the part of the call nothing overlaps, so it should be short), and the rest is cut in two."""
    global _sm_count
    if _sm_count is None:
        _sm_count = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    sm = _sm_count
    waves = lambda e: -(-ctas_of(e) // sm) if e > 0 else 0

    def cap(w):                                                  # most envs whose grid fits in w waves
        lo, hi = 0, n_envs
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if waves(mid) <= w else (lo, mid - 1)
        return lo

    total = waves(n_envs)
    if total <= 2:
        return [n_envs]
    rest = cap(total - 1)                                        # fills total - 1 waves; the tail goes last
    if rest <= 0 or rest >= n_envs:
        return [n_envs]
    first = cap((total - 1 + 1) // 2)
    if 0 < first < rest and waves(first) + waves(rest - first) + waves(n_envs - rest) <= total:
        return [first, rest, n_envs]
    return [rest, n_envs]


def as_host(x, dtype=torch.float32):
    """numpy / CPU tensor -> CPU tensor of `dtype` (shares memory when no conversion is needed)."""
    import numpy as np
    t = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
    assert not t.is_cuda
    return t.to(dtype)


def layout(kind, *dims):
    """(total floats per agent, [offsets]) of a flat parameter buffer."""
    n = {"gat": 20, "beh": 8, "actor": 22, "critic": 26, "pdec": 8, "bdec": 8, "bfc": 6, "bfcdec": 6}[kind]
    arr = (C.c_int64 * n)()
    fn = getattr(lib, f"iplan_{kind}_layout")
    total = fn(*dims, C.cast(arr, C.c_void_p))
    return int(total), [int(x) for x in arr]
