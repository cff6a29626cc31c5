"""The hard-update behaviour module (iPLAN-Hard ablation, iplan_b200/nova/behavior_policy.py) on the GPU: ``learn``
against the reference's recorded call and the oracle, ``latent_update`` against the reference's recorded calls, the
runner wiring, checkpoints, and the shapes it rejects."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _check():
    import importlib
    return importlib.import_module("tools.check_beh_learn_hard")


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_hard_learn_vs_reference_golden(case):
    """One recorded ``learn`` call of the reference's nova/behavior_policy (same dropout masks): per-agent losses 1e-4
    relative, every clipped gradient tensor 1e-3 relative to the oracle, post-step weights 1e-6 from the reference's.
    The highway case has 110 chains per agent-net: a full 64-chain tile and a ragged one."""
    _need_gpu()
    assert _check().run(case)


def test_hard_learn_bench_shape_vs_oracle():
    """A=5, N=55, B=8, T=90 (440 chains per agent-net: six full tiles and a ragged one; 8 trained windows), agents
    terminating inside the episode, dropout replayed: against the oracle from the same weights."""
    _need_gpu()
    chk = _check()
    from tools.check_beh_learn_tile import make_batch
    from iplan_b200.config import make_args
    from iplan_b200.nova.behavior_policy import Behavior_policy
    args = make_args("highway", use_cuda=True, device="cuda", soft_update_enable=False)
    A, N, W, B, T = args.n_agents, args.max_vehicle_num, args.max_history_len, 8, 90
    assert A == 5 and N == 55
    batch = make_batch(args, B, T + 1, seed=21)
    n_pos = T // W - 1
    gen = torch.Generator().manual_seed(22)
    keeps = [torch.rand(n_pos, B * N, W, args.decoder_rnn_dim, generator=gen) >= args.decoder_dropout for _ in range(A)]
    torch.manual_seed(23)
    pol = Behavior_policy(args, None)
    enc_before = [{k: v.detach().cpu().clone() for k, v in n.state_dict().items()} for n in pol.behavior_encoder]
    dec_before = [{k: v.detach().cpu().clone() for k, v in n.state_dict().items()} for n in pol.behavior_decoder]
    pol.debug_keep = chk.keep_for_gpu(keeps, B, N, W)
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    data = {"history": batch["history"].cpu(), "terminated": batch["terminated"].cpu()}
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    assert chk.compare(pol, data, keeps, oargs, enc_before, dec_before, losses, tag="B=8 T=90")


def _latent_policy(g):
    from iplan_b200.config import make_args
    from iplan_b200.nova.behavior_policy import Behavior_policy
    args = make_args(g["args"]["env"], use_cuda=True, device="cuda")
    for k, v in g["args"].items():
        setattr(args, k, v)
    args.use_cuda, args.device = True, "cuda"
    pol = Behavior_policy(args, None)
    for a, sd in enumerate(g["enc_after"]):
        pol.behavior_encoder[a].load_state_dict(sd)
    return pol


@pytest.mark.parametrize("case", ["mpe", "highway"])
@pytest.mark.parametrize("large", [False, True])
def test_hard_latent_update_vs_reference_golden(case, large):
    """Three consecutive ``latent_update`` calls (hidden state carried, prev_latent random) against the reference's hard
    module; ``large`` repeats the recorded envs to >= PIPELINE_MIN_ROWS so that the pipelined native path runs.  The
    result does not depend on prev_latent at all: K1b with coefficient 1 gives the encoder's soft-max output bit for bit."""
    _need_gpu()
    from iplan_b200 import _lib
    chk = _check()
    g = chk.load_case(case)
    pol = _latent_policy(g)
    steps = g["latent_steps"]
    B0 = steps[0]["window"].shape[0]
    reps = -(-_lib.PIPELINE_MIN_ROWS // B0) if large else 1
    tile = lambda x: np.ascontiguousarray(np.concatenate([np.asarray(x)] * reps, axis=0))
    hid = tile(steps[0]["hid_in"].numpy())
    rng = np.random.default_rng(4)
    for t, st in enumerate(steps):
        window, prev = tile(st["window"].numpy()), tile(st["prev"].numpy())
        other = (rng.standard_normal(prev.shape) * 1e30).astype(np.float32)        # any finite prev_latent
        lat2, _ = pol.latent_update(window, hid.copy() if isinstance(hid, np.ndarray) else hid.clone(), other)
        lat, hid = pol.latent_update(window, hid, prev)
        torch.cuda.synchronize()
        assert np.array_equal(np.asarray(lat), np.asarray(lat2)), t
        assert torch.is_tensor(hid) and tuple(hid.shape) == tuple(tile(st["hid_out"].numpy()).shape)
        dl = float(np.abs(np.asarray(lat) - tile(st["latent"].numpy())).max())
        dh = float(np.abs(hid.cpu().numpy() - tile(st["hid_out"].numpy())).max())
        print(f"[latent_update hard {case} B={B0 * reps} step {t}] latent {dl:.2e} hidden {dh:.2e}")
        assert dl < 1e-5 and dh < 1e-5


def test_hard_module_in_runner_device_equals_reference_api():
    """build_system(soft_update_enable=False) wires the hard module; the device-resident runner and the reference's call
    pattern (latent_update every timestep) then store the same episode, and ``learn`` trains on it."""
    _need_gpu()
    from iplan_b200.nova.behavior_policy import Behavior_policy
    from iplan_b200.runners.synthetic_runner import build_system
    kw = dict(n_envs=24, env="highway", hazard=0.002, seed=9, episode_limit=30, soft_update_enable=False)
    sa, sb = build_system(**kw), build_system(**kw)
    assert isinstance(sa.behavior, Behavior_policy) and isinstance(sb.behavior, Behavior_policy)
    assert sa.behavior.soft_update_coef == 1.0
    assert torch.equal(sa.behavior.stack.flat, sb.behavior.stack.flat)
    ba, *_ = sa.runner.run(test_mode=True)
    bb, *_ = sb.runner.run_reference_api(test_mode=True)
    torch.cuda.synchronize()
    T = sa.args.episode_limit
    assert torch.equal(ba["actions"][:, :T], bb["actions"][:, :T])
    for key in ("attention_latent", "behavior_latent", "history", "rnn_states_actors", "rnn_states_critics"):
        d = float((ba[key].float() - bb[key].float()).abs().max())
        print(f"[hard runner vs api] {key}: {d:.3e}")
        assert d <= 1e-6, (key, d)
    losses = sa.behavior.learn(ba, t_env=0)
    assert len(losses) == sa.args.n_agents and all(np.isfinite(float(x)) and float(x) > 0 for x in losses)
    assert set(sa.behavior.train_info) == {"behavior_loss", "behavior_encoder_grad_norm", "behavior_decoder_grad_norm"}
    # build_system keeps the soft module by default
    from iplan_b200.nova import stable_behavior_policy
    assert type(build_system(n_envs=4, env="highway", episode_limit=30).behavior) is stable_behavior_policy.Behavior_policy


def test_hard_checkpoint_and_optimiser_round_trip(tmp_path):
    """save_models / load_models(load_optimisers=True) after one ``learn``: weights and Adam state come back exactly, and
    ``behavior_optimizer_{i}_opt.th`` loads into torch.optim.Adam over the encoder then decoder tensors."""
    _need_gpu()
    chk = _check()
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.nova.behavior_policy import Behavior_policy
    from tools.check_pred_learn import scheme_for
    g = chk.load_case("mpe")
    args = chk.gpu_args(g)
    d = g["data"]
    B, T1 = d["history"].shape[:2]
    scheme, groups, pre = scheme_for(args)
    batch = EpisodeBatch(scheme, groups, B, T1, preprocess=pre, device="cuda")
    batch.update({k: v.numpy() for k, v in d.items()}, bs=slice(None), ts=slice(None))
    pol = Behavior_policy(args, None)
    pol.learn(batch, t_env=0)
    pol.save_models(str(tmp_path))
    for i in range(args.n_agents):
        for f in (f"behavior_encoder_{i}.th", f"behavior_decoder_{i}.th", f"behavior_optimizer_{i}_opt.th"):
            assert os.path.exists(tmp_path / f), f
    back = Behavior_policy(args, None)
    back.load_models([str(tmp_path)], load_optimisers=True)
    assert torch.equal(back.stack.flat, pol.stack.flat) and torch.equal(back.dec_stack.flat, pol.dec_stack.flat)
    ws, wb = pol._learn_state(), back._learn_state()
    assert wb["step"] == ws["step"] == 1
    for k in ("m_enc", "v_enc", "m_dec", "v_dec"):
        assert torch.equal(wb[k], ws[k]), k
    sd = torch.load(tmp_path / "behavior_optimizer_1_opt.th", weights_only=False)
    params = [torch.nn.Parameter(torch.zeros(shape)) for _, shape in pol.stack.spec + pol.dec_stack.spec]
    opt = torch.optim.Adam(params, lr=args.lr_behavior, eps=args.optim_eps)
    opt.load_state_dict(sd)
    off, shape = pol.dec_stack.named_offsets()["decoder.rnn.weight_hh_l0"]
    pid = len(pol.stack.spec) + [n for n, _ in pol.dec_stack.spec].index("decoder.rnn.weight_hh_l0")
    n = int(np.prod(shape))
    assert torch.equal(opt.state[params[pid]]["exp_avg"], ws["m_dec"][1, off:off + n].view(shape).cpu())


def test_hard_learn_rejects_partial_and_short_episodes():
    """T % W != 0 raises (the reference's reshape does, verified at T = 25), and so does T < 2 W (no window to predict);
    the native entry point rejects a geometry whose targets leave the episode, before any launch."""
    _need_gpu()
    from iplan_b200 import _lib
    from iplan_b200.nova.behavior_policy import Behavior_policy
    from tools.check_beh_learn_tile import make_batch
    from iplan_b200.config import make_args
    args = make_args("highway", use_cuda=True, device="cuda", soft_update_enable=False)
    pol = Behavior_policy(args, None)
    before = pol.stack.flat.clone()
    for T in (25, 10, 15):
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError):
            pol.learn(make_batch(args, 2, T + 1, seed=1), t_env=0)
        assert _lib.launch_count() == n0
    assert torch.equal(pol.stack.flat, before)
    z = torch.zeros(64, device="cuda")
    p = _lib.ptr(z)
    W = args.max_history_len
    for n_pos, step, first in ((2, W, 0 + 1), (3, W, 0), (1, W, -W - 1), (0, W, 0), (2, 0, 0)):
        n0 = _lib.launch_count()
        rc = _lib.lib.iplan_beh_learn_windows(p, 64, p, 64, p, p, p, p, p, None, p, p, p, 64, 1, 0, 0.1, 1.0, 0.0,
                                              1, 1, 3 * W, 1, 5, 8, W, n_pos, step, first, _lib.stream())
        assert rc != 0 and _lib.launch_count() == n0, (n_pos, step, first)
        assert b"beh_learn_windows" in _lib.lib.iplan_last_error()
