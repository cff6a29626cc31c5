"""The fully-connected behaviour module (iPLAN-FC ablation, iplan_b200/nova/behavior_FC_policy.py) on the GPU: ``learn``
against the reference's recorded calls and the float64 oracle, bit-for-bit repeatability, ``latent_update`` against the
reference's recorded calls, the time-strided rollout step, the runner wiring, and checkpoints."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _case(case):
    if GOLDEN not in sys.path:
        sys.path.insert(0, GOLDEN)
    from beh_fc_inputs import load_fc_case
    return load_fc_case(GOLDEN, case)


def _args(g):
    from iplan_b200.config import make_args
    args = make_args(g["args"].get("env", "highway"))
    for k, v in g["args"].items():
        setattr(args, k, v)
    args.use_cuda, args.device = True, "cuda"
    return args


def _batch(args, data):
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from tools.check_pred_learn import scheme_for
    B, T1 = data["history"].shape[:2]
    scheme, groups, pre = scheme_for(args)
    batch = EpisodeBatch(scheme, groups, B, T1, preprocess=pre, device="cuda")
    batch.update({k: v.numpy() for k, v in data.items()}, bs=slice(None), ts=slice(None))
    return batch


def _policy(args, enc=None, dec=None):
    from iplan_b200.nova.behavior_FC_policy import Behavior_policy
    pol = Behavior_policy(args, None)
    for a in range(args.n_agents):
        if enc is not None:
            pol.behavior_encoder[a].load_state_dict(enc[a])
        if dec is not None:
            pol.behavior_decoder[a].load_state_dict(dec[a])
    return pol


def _bench_shape_args():
    from iplan_b200.config import make_args
    return make_args("highway", use_cuda=True, device="cuda", behavior_fully_connected=True)


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_fc_learn_vs_reference_golden(case):
    """One recorded ``learn`` call of the reference's nova/behavior_FC_policy: per-agent losses 1e-5 relative, post-step
    weights 1e-6 from the reference's.  The highway case has 2090 rows per agent-net: 32 full 64-row tiles and a ragged
    one of 42 rows."""
    _need_gpu()
    g = _case(case)
    args = _args(g)
    pol = _policy(args, g["enc_before"], g["dec_before"])
    b_loss, s_loss, t_loss = pol.learn(_batch(args, g["data"]), t_env=0)
    torch.cuda.synchronize()
    assert s_loss == [] and len(b_loss) == len(t_loss) == args.n_agents
    for a in range(args.n_agents):
        rel = abs(float(b_loss[a]) - g["behavior_loss"][a]) / abs(g["behavior_loss"][a])
        worst = max(max(float((v.cpu() - g["enc_after"][a][k]).abs().max()) for k, v in pol.behavior_encoder[a].state_dict().items()),
                    max(float((v.cpu() - g["dec_after"][a][k]).abs().max()) for k, v in pol.behavior_decoder[a].state_dict().items()))
        print(f"[fc learn {case} a={a}] loss rel {rel:.2e}, max |weight - reference| after the step {worst:.2e}")
        assert rel <= 1e-5 and worst <= 1e-6
        assert float(t_loss[a]) == float(b_loss[a])
    assert set(pol.train_info) == {"behavior_loss", "stability_loss", "behavior_total", "behavior_encoder_grad_norm",
                                   "behavior_decoder_grad_norm"}
    assert abs(pol.train_info["behavior_loss"] - g["stats"][[k for k in g["stats"] if k.endswith("behavior_loss")][0]]) \
        <= 1e-5 * abs(pol.train_info["behavior_loss"])


def test_fc_learn_bench_shape_vs_float64_oracle():
    """A=5, N=55, B=8, T=90 (79 positions, 34760 rows per agent-net, a ragged last tile): loss 1e-6 relative and every raw
    gradient tensor 1e-5 relative to the float64 oracle run from the same weights."""
    _need_gpu()
    from tools.beh_fc_oracle import behavior_learn_fc_agent
    from tools.check_beh_learn_tile import make_batch
    args = _bench_shape_args()
    A, N, B, T = args.n_agents, args.max_vehicle_num, 8, 90
    batch = make_batch(args, B, T + 1, seed=31)
    torch.manual_seed(32)
    pol = _policy(args)
    enc0 = [{k: v.detach().cpu().double() for k, v in n.state_dict().items()} for n in pol.behavior_encoder]
    dec0 = [{k: v.detach().cpu().double() for k, v in n.state_dict().items()} for n in pol.behavior_decoder]
    b_loss, _, _ = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    hist = batch["history"][:, :-1].cpu().double()
    term = batch["terminated"][:, :-1, :, 0].cpu().double()
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    for a in range(A):
        ref, _ = behavior_learn_fc_agent(enc0[a], dec0[a], hist[:, :, a], term[:, :, a], oargs)
        rel = abs(float(b_loss[a]) - ref["behavior_loss"]) / abs(ref["behavior_loss"])
        assert rel <= 1e-6, (a, rel)
        worst = 0.0
        for kind, stack in (("enc", pol.stack), ("dec", pol.dec_stack)):
            for name, (off, shape) in stack.named_offsets().items():
                n = int(np.prod(shape))
                mine = pol.last_grads[kind][a, off:off + n].view(shape).cpu().double()
                want = ref["grads"][kind + ":" + name]
                r = float((mine - want).abs().max() / want.abs().max())
                worst = max(worst, r)
                assert r <= 1e-5, (a, kind, name, r)
        print(f"[fc learn B=8 T=90 a={a}] loss rel {rel:.2e}, worst gradient tensor rel {worst:.2e}")


def test_fc_learn_is_bit_repeatable_and_ignores_terminated():
    """Two calls from the same state give the same bits (the cross-CTA sums are added in a fixed order), and so does a
    batch that differs only in ``terminated``."""
    _need_gpu()
    from tools.check_beh_learn_tile import make_batch
    args = _bench_shape_args()
    batch = make_batch(args, 8, 91, seed=41)
    other = make_batch(args, 8, 91, seed=41)
    other["terminated"][:] = 1 - other["terminated"]
    assert not torch.equal(batch["terminated"], other["terminated"])
    out = []
    for b in (batch, batch, other):
        torch.manual_seed(42)
        pol = _policy(args)
        loss, _, _ = pol.learn(b, t_env=0)
        out.append((loss, pol.last_grads, pol.stack.flat.clone(), pol.dec_stack.flat.clone()))
    for loss, grads, enc, dec in out[1:]:
        assert [float(x) for x in loss] == [float(x) for x in out[0][0]]
        assert torch.equal(grads["enc"], out[0][1]["enc"]) and torch.equal(grads["dec"], out[0][1]["dec"])
        assert torch.equal(enc, out[0][2]) and torch.equal(dec, out[0][3])


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_fc_latent_update_vs_reference_golden(case):
    """Three ``latent_update`` calls of the reference's FC module with the trained encoder: latent within 1e-6, the
    hidden state handed back unchanged, prev_latent ignored, the result a read-only array."""
    _need_gpu()
    g = _case(case)
    pol = _policy(_args(g), g["enc_after"])
    for t, st in enumerate(g["latent_steps"]):
        window = st["window"].numpy()
        hid = object()
        lat, hid_out = pol.latent_update(window, hid, np.full(st["latent"].shape, 1e30, dtype=np.float32))
        assert hid_out is hid and not lat.flags.writeable
        d = float(np.abs(lat - st["latent"].numpy()).max())
        print(f"[fc latent_update {case} step {t}] {d:.2e}")
        assert d < 1e-6


def test_fc_strided_step_equals_explicit_window():
    """The rollout reads windows in place from the time-strided episode store (win_stride_step, win_pad); that gives the
    same bits as the explicit [A,B,N,W*o] window, at every padding the episode start produces."""
    _need_gpu()
    args = _bench_shape_args()
    A, N, o, W, L, B, T = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.max_history_len, args.latent_dim, 6, 14
    torch.manual_seed(3)
    pol = _policy(args)
    store = torch.rand(B, T, A, N, o, device="cuda") * 2 - 1            # [B, T, A, N, o]: the runner's history store
    src = store.permute(1, 2, 0, 3, 4)                                   # [T, A, B, N, o] view
    for t in range(T):
        first, pad = max(0, t - W + 1), max(0, W - 1 - t)
        win = torch.zeros(A, B, N, W, o, device="cuda")
        win[:, :, :, pad:] = store[:, first:t + 1].permute(2, 0, 3, 1, 4)
        a_out = torch.empty(A, B, N, L, device="cuda")
        b_out = torch.full((A, B, N, L), float("nan"), device="cuda")
        pol.behavior_step(win.reshape(A, B, N, W * o), None, None, a_out)
        pol.behavior_step(src[first], None, None, b_out, win_stride_step=store.stride(1), win_pad=pad)
        torch.cuda.synchronize()
        assert torch.equal(a_out, b_out), t


def test_fc_module_in_runner_device_equals_reference_api():
    """build_system(behavior_fully_connected=True) wires the FC module even with soft_update_enable; the device-resident
    runner and the reference's call pattern (latent_update every timestep) store the same episode, and ``learn`` trains
    on it."""
    _need_gpu()
    from iplan_b200.nova.behavior_FC_policy import Behavior_policy
    from iplan_b200.runners.synthetic_runner import build_system
    kw = dict(n_envs=24, env="highway", hazard=0.002, seed=9, episode_limit=30, behavior_fully_connected=True)
    sa, sb = build_system(**kw), build_system(**kw)
    assert type(sa.behavior) is Behavior_policy and sa.args.soft_update_enable
    assert torch.equal(sa.behavior.stack.flat, sb.behavior.stack.flat)
    ba, *_ = sa.runner.run(test_mode=True)
    bb, *_ = sb.runner.run_reference_api(test_mode=True)
    torch.cuda.synchronize()
    T = sa.args.episode_limit
    assert torch.equal(ba["actions"][:, :T], bb["actions"][:, :T])
    for key in ("attention_latent", "behavior_latent", "history", "rnn_states_actors", "rnn_states_critics"):
        d = float((ba[key].float() - bb[key].float()).abs().max())
        print(f"[fc runner vs api] {key}: {d:.3e}")
        assert d <= 1e-6, (key, d)
    assert float(ba["behavior_latent"][:, 1:T].abs().sum()) > 0
    losses, stab, _ = sa.behavior.learn(ba, t_env=0)
    assert stab == [] and all(np.isfinite(float(x)) and float(x) > 0 for x in losses)


def test_fc_checkpoint_and_optimiser_round_trip(tmp_path):
    """save_models / load_models(load_optimisers=True) after one ``learn``: weights and Adam state come back exactly; the
    files carry the key names and shapes the reference's own files have (recorded in the fixture), and
    ``behavior_optimizer_{i}_opt.th`` loads into torch.optim.Adam over the encoder then decoder tensors."""
    _need_gpu()
    g = _case("highway")
    args = _args(g)
    pol = _policy(args, g["enc_before"], g["dec_before"])
    pol.learn(_batch(args, g["data"]), t_env=0)
    pol.save_models(str(tmp_path))
    files = g["files"]
    enc_sd = torch.load(tmp_path / "behavior_encoder_0.th", weights_only=False)
    dec_sd = torch.load(tmp_path / "behavior_decoder_0.th", weights_only=False)
    opt_sd = torch.load(tmp_path / "behavior_optimizer_0_opt.th", weights_only=False)
    assert [(k, tuple(v.shape)) for k, v in enc_sd.items()] == [tuple(e) for e in files["encoder"]]
    assert [(k, tuple(v.shape)) for k, v in dec_sd.items()] == [tuple(e) for e in files["decoder"]]
    assert {pid: tuple(s["exp_avg"].shape) for pid, s in opt_sd["state"].items()} == files["optimizer"]
    assert list(opt_sd["param_groups"][0]["params"]) == files["optimizer_params"]
    back = _policy(args)
    back.load_models([str(tmp_path)], load_optimisers=True)
    assert torch.equal(back.stack.flat, pol.stack.flat) and torch.equal(back.dec_stack.flat, pol.dec_stack.flat)
    ws, wb = pol._learn_state(), back._learn_state()
    assert wb["step"] == ws["step"] == 1
    for k in ("m_enc", "v_enc", "m_dec", "v_dec"):
        assert torch.equal(wb[k], ws[k]), k
    params = [torch.nn.Parameter(torch.zeros(shape)) for _, shape in pol.stack.spec + pol.dec_stack.spec]
    opt = torch.optim.Adam(params, lr=args.lr_behavior, eps=args.optim_eps)
    opt.load_state_dict(torch.load(tmp_path / "behavior_optimizer_1_opt.th", weights_only=False))
    off, shape = pol.dec_stack.named_offsets()["decoder.linear_2.weight"]
    pid = len(pol.stack.spec) + [n for n, _ in pol.dec_stack.spec].index("decoder.linear_2.weight")
    n = int(np.prod(shape))
    assert torch.equal(opt.state[params[pid]]["exp_avg"], ws["m_dec"][1, off:off + n].view(shape).cpu())


def test_fc_learn_rejects_short_episodes():
    """n_pos = T - 1 - W < 1 raises before any launch (the reference divides by zero there) and leaves the weights."""
    _need_gpu()
    from iplan_b200 import _lib
    from tools.check_beh_learn_tile import make_batch
    args = _bench_shape_args()
    pol = _policy(args)
    before = pol.stack.flat.clone()
    W = args.max_history_len
    for T in (W + 1, W):
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError):
            pol.learn(make_batch(args, 2, T + 1, seed=1), t_env=0)
        assert _lib.launch_count() == n0
    assert torch.equal(pol.stack.flat, before)
