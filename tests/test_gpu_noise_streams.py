"""The kernels' own noise: every kernel that draws Philox noise runs its production path (no explicit noise), and
oracle/philox.py replays the draws — Gumbel noise, sampling uniforms, dropout masks — into the float64 oracle or into the
kernel's explicit-noise argument.  A wrong key, counter, word index or layout in a kernel, a dropout mask that two
launches draw differently, or pipelined chunks that reuse a counter make these comparisons fail.

Tolerances.  Outputs of the rollout kernels: 1e-4 (as the explicit-noise parity tests).  Learner gradients, per tensor:
1e-5 relative to the tensor's largest entry, or, where float32 arithmetic itself is less accurate than that, 3x the
distance of the float32 oracle from the float64 oracle on the same inputs; every margin is printed."""
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOL = 1e-4
GRAD_REL = 1e-5
# The soft behaviour learner's encoder GRU weight gradients sum about 350 000 terms per entry (440 chains x 79 window
# positions x 10 steps) in long float32 register sums before the atomics; at this shape they were measured 1.6e-6 to
# 2.0e-5 from float64 on an NVIDIA H100 80GB HBM3 (400 W), against 5e-7 to 1e-6 for the float32 oracle's autograd.  Their
# floor is 5e-5; a wrong dropout draw or window moves them by far more.
ENC_GRU_FLOOR = {"enc:rnn.weight_ih_l0": 5e-5, "enc:rnn.weight_hh_l0": 5e-5}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _params(nets, dtype=torch.float32):
    return [{k: v.detach().cpu().to(dtype).clone() for k, v in n.state_dict().items()} for n in nets]


def _rel(x, ref):
    x, ref = x.double(), ref.double()
    return float((x - ref).abs().max() / (ref.abs().max() + 1e-30))


def _bound(spread32):
    return max(GRAD_REL, 3.0 * spread32)


def _absdiff(x, ref):
    return float((x.double() - ref.double()).abs().max())


def _check_tensors(tag, mine, o64, o32, absolute=False, floors=None):
    """mine / o64 / o32: {name: tensor}.  Each tensor within max(1e-5 relative to its largest entry, 3 x the float32
    oracle's distance) of the float64 oracle.  ``absolute``: post-step weights, max(1e-6, 3 x the float32 oracle's
    distance) in absolute terms (one Adam step moves a weight by about the learning rate whatever its size).
    ``floors``: {name: a larger floor} for tensors whose documented accuracy is below 1e-5."""
    bad = []
    diff, floor = (_absdiff, 1e-6) if absolute else (_rel, GRAD_REL)
    for name, want in o64.items():
        rel, spread = diff(mine[name], want), diff(o32[name], want)
        bound = max((floors or {}).get(name, floor), 3.0 * spread)
        ok = rel <= bound
        print(f"    {tag} {name:34s} cuda {rel:.2e}  fp32 oracle {spread:.2e}  bound {bound:.2e}{'' if ok else '   <-- FAIL'}")
        if not ok:
            bad.append(name)
    return bad


def _gat_inputs(B, A, N, o, L, D, seed=3):
    rng = np.random.default_rng(seed)
    hist = rng.uniform(-1, 1, size=(B, A, N, o)).astype(np.float32)
    hist[..., 0] = 1.0
    hist[:, :, 30:] = 0.0
    beh = rng.dirichlet(np.ones(L), size=(B, A, N)).astype(np.float32)
    att = rng.uniform(-1, 1, size=(B, A, N, D)).astype(np.float32)
    return hist, att, beh


def _gat_oracle64(params, hist, att, beh, gum):
    """O.gat_forward per agent-net in float64: (out [B, A, N, D], hard gates [A, B, N, N-1])."""
    from oracle import iplan_oracle as O
    B, A, N, _ = hist.shape
    outs, hards = [], []
    for a in range(A):
        p = {k: v.double() for k, v in params[a].items()}
        x = torch.cat([torch.as_tensor(hist[:, a]), torch.as_tensor(beh[:, a])], dim=-1).double()
        h, parts = O.gat_forward(p, x, torch.as_tensor(att[:, a]).double().reshape(B * N, -1), torch.as_tensor(gum[a]).double(),
                                 return_parts=True)
        outs.append(h.view(B, 1, N, -1))
        hards.append(parts["hard"])
    return torch.cat(outs, dim=1), torch.stack(hards)


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [6, 3])
def test_k1_philox_direct_path_vs_oracle(B):
    """K1 drawing its own Gumbel noise (direct path, hard gates captured) against the float64 oracle fed the replay."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from oracle import philox as PX
    args = make_args("highway")
    A, N, o, L, D = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim
    torch.manual_seed(5)
    pred = Prediction_policy(args, None)
    params = _params(pred.pred_GAT)
    hist, att, beh = _gat_inputs(B, A, N, o, L, D)
    pred.calls = 17                                           # any counter: the replay must follow it
    pred.capture_hard = True
    out = pred.GAT_latent_update(hist, att, beh)
    assert pred.calls == 18
    hard = pred.last_hard.cpu().double()
    gum = PX.gat_step_gumbel(pred.seed, 17, A, B, N)
    ref, ref_hard = _gat_oracle64(params, hist, att, beh, gum)
    d = float((torch.as_tensor(out).double() - ref).abs().max())
    mid = (ref_hard > 0.01) & (ref_hard < 0.99)
    dh = (hard - ref_hard).abs()
    print(f"[K1 philox B={B}] max |out - oracle64| {d:.3e}; hard gates: max diff {float(dh.max()):.3e} overall, "
          f"{float(dh[~mid].max()):.3e} on well-conditioned gates, {float(dh[mid].max()) if mid.any() else 0.0:.3e} on the "
          f"ill-conditioned fraction {float(mid.double().mean()):.4f} (oracle gate in (0.01, 0.99))")
    assert d < TOL
    assert float(dh.max()) < 1e-3                             # a wrong draw moves a gate by O(1)


def test_k1_philox_pipelined_chunks_vs_oracle():
    """The native pipelined GAT_latent_update at 130 envs: chunk c draws with counter calls + c over its own envs.  Envs
    at both ends of every chunk against the float64 oracle fed the per-chunk replay."""
    _need_gpu()
    from iplan_b200 import _lib
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from oracle import philox as PX
    args = make_args("highway", use_cuda=True, device="cuda")
    B, A, N, o, L, D = 130, args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim
    assert B >= _lib.PIPELINE_MIN_ROWS
    torch.manual_seed(11)
    pred = Prediction_policy(args, None)
    params = _params(pred.pred_GAT)
    hist, att, beh = _gat_inputs(B, A, N, o, L, D, seed=4)
    ends = _lib.wave_chunks(B, lambda e: (2 * e * A + 3) // 4)
    assert len(ends) >= 2, ends
    c0 = pred.calls
    out = pred.GAT_latent_update(hist, att, beh)
    assert pred.calls - c0 == len(ends)
    S = sorted({0, B - 1} | {e for e in ends[:-1]} | {e - 1 for e in ends})
    gum = PX.gat_latent_update_gumbel(pred.seed, c0, A, ends, N)[:, S]
    ref, _ = _gat_oracle64(params, hist[S], att[S], beh[S], gum)
    d = float((torch.as_tensor(out[S]).double() - ref).abs().max())
    print(f"[K1 pipelined, chunk ends {ends}] envs {S}: max |out - oracle64| {d:.3e}")
    assert d < TOL


# ------------------------------------------------------------------------------------------------------------------------
def _controller(B, seed=8):
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.config import make_args
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from tests.test_gpu_rollout import make_scheme
    args = make_args("highway")
    args.use_cuda, args.device = True, "cuda"
    scheme, groups, pre = make_scheme(args)
    batch = EpisodeBatch(scheme, groups, 1, 2, preprocess=pre, device="cuda")
    torch.manual_seed(seed)
    mac = DcntrlMAC(batch.scheme, groups, args)
    A, F = args.n_agents, mac.input_shape
    rng = np.random.default_rng(seed)
    feat = torch.tensor(rng.uniform(-1, 1, size=(A, B, F)).astype(np.float32)).cuda()
    ra = torch.tensor(rng.uniform(-1, 1, size=(A, B, 64)).astype(np.float32)).cuda()
    rc = torch.tensor(rng.uniform(-1, 1, size=(A, B, 64)).astype(np.float32)).cuda()
    return args, mac, feat, ra, rc


def _ctrl_run(mac, feat, ra, rc, avail, uniforms):
    A, B = feat.shape[:2]
    na, nc = torch.empty(A, B, 64, device="cuda"), torch.empty(A, B, 64, device="cuda")
    logits = torch.empty(A, B, mac.args.n_actions, device="cuda")
    act, lp, val = mac.controller_step(feat, ra, rc, na, nc, avail, test_mode=False, uniforms=uniforms, logits=logits)
    torch.cuda.synchronize()
    return [x.clone() for x in (act, lp, val, na, nc, logits)]


def test_k1c_philox_sampling_equals_replayed_uniforms():
    """K1c drawing its own uniforms, then again with the replayed uniforms passed explicitly: bit-equal actions,
    log-probs, values and hidden states."""
    _need_gpu()
    from oracle import philox as PX
    B = 300
    args, mac, feat, ra, rc = _controller(B)
    A, nA = args.n_agents, args.n_actions
    with torch.no_grad():
        for net in mac.agents:
            net.act.action_out.linear.weight.mul_(30.0)
    avail = torch.ones(A, B, nA, dtype=torch.uint8, device="cuda")
    avail[:, ::7, 1] = 0
    mac.calls = 41
    got = _ctrl_run(mac, feat, ra, rc, avail, None)
    uni = torch.as_tensor(PX.controller_uniforms(mac.seed, 41, A, B)).cuda()
    again = _ctrl_run(mac, feat, ra, rc, avail, uni)
    names = ("actions", "logp", "values", "rnn_a", "rnn_c", "logits")
    for n, x, y in zip(names, got, again):
        assert torch.equal(x, y), n
    counts = torch.bincount(got[0].view(-1).long(), minlength=nA).tolist()
    print(f"[K1c philox] {A * B} samples bit-equal to the replay; action counts {counts}")
    assert len(set(counts)) > 1 and min(counts) > 0


def test_k1c_sampler_never_returns_an_unavailable_action():
    """Explicit uniforms at the edges of the range — the smallest and the largest u01, 1.0 and the fp32 values just above the
    sampler's last cdf — on agent-nets whose logits are set exactly (head weight 0, bias = the logits): the last action
    masked; the first and the last two masked; an available last action whose probability underflows to 0; a zero-
    probability action in the middle with the last one masked; nothing masked.  The chosen action must be available, have
    probability > 0 and equal the float64 inverse-CDF choice (at the top of the range: the last action with probability
    > 0)."""
    _need_gpu()
    from iplan_b200.config import make_args
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    nA = make_args("highway").n_actions
    assert nA == 5
    base = [0.1, 0.3, -0.2, 0.5, 0.0]
    cases = [  # (bias, avail)
        (base, [1, 1, 1, 1, 0]),
        (base, [0, 1, 1, 0, 0]),
        (base[:4] + [-1000.0], [1, 1, 1, 1, 1]),
        (base[:2] + [-1000.0] + base[3:], [1, 1, 1, 1, 0]),
        (base, [1, 1, 1, 1, 1]),
    ]
    A = len(cases)
    # the kernel's fp32 probabilities and inclusive scan (lane shuffles at offsets 1, 2, 4), emulated to find its last cdf
    tops = []
    for bias, av in cases:
        lg = np.where(np.array(av) == 0, np.float32(-1e10), np.array(bias, dtype=np.float32)).astype(np.float32)
        ex = np.exp((lg - lg.max()).astype(np.float32)).astype(np.float32)
        pr = np.exp((lg - lg.max() - np.log(ex.sum(dtype=np.float32))).astype(np.float32)).astype(np.float32)
        cdf = pr.copy()
        for off in (1, 2, 4):
            cdf = np.concatenate([cdf[:off], (cdf[off:] + cdf[:-off]).astype(np.float32)])
        tops.append(np.float32(cdf[-1]))
    us = {PX.u01(0), PX.u01(0xFFFFFFFF), np.float32(1 - 2.0 ** -23), np.float32(1.0)}
    for t in tops:
        x = t
        for _ in range(3):
            x = np.nextafter(x, np.float32(2))
            us.add(np.float32(min(x, np.float32(1.0))))
    us = sorted(us)
    B = len(us)
    args, mac, feat, ra, rc = _controller(B, seed=9)
    assert args.n_agents == A
    with torch.no_grad():
        for a, (bias, _) in enumerate(cases):
            mac.agents[a].act.action_out.linear.weight.zero_()
            mac.agents[a].act.action_out.linear.bias.copy_(torch.tensor(bias))
    avail = torch.tensor([av for _, av in cases], dtype=torch.uint8).view(A, 1, nA).expand(A, B, nA).contiguous().cuda()
    uni = torch.tensor(np.array(us, dtype=np.float32)).view(1, B).expand(A, B).contiguous().cuda()
    act, lp, _, _, _, logits = _ctrl_run(mac, feat, ra, rc, avail, uni)
    act = act.cpu().long()
    for a, (bias, av) in enumerate(cases):
        lg64 = torch.where(torch.tensor(av) == 0, torch.tensor(-1e10, dtype=torch.float64), torch.tensor(bias, dtype=torch.float64))
        assert torch.equal(logits[a, 0].cpu(), lg64.float()), (a, logits[a, 0])       # the logits are exactly the bias
        p64 = torch.softmax(lg64, -1).expand(B, nA)
        want = O.inverse_cdf(p64, torch.tensor(np.array(us, dtype=np.float64)))
        print(f"[K1c edges] case {a}: avail {av}, p64 {[f'{float(p):.3g}' for p in p64[0]]}, fp32 last cdf {float(tops[a]):.9g}: "
              f"actions {act[a].tolist()} expected {want.tolist()}")
        for b in range(B):
            k = int(act[a, b])
            assert av[k] == 1 and float(p64[0, k]) > 0.0, (a, float(us[b]), k)
            assert k == int(want[b]), (a, float(us[b]), k, int(want[b]))
        assert torch.isfinite(lp[a]).all() and float(lp[a].min()) > -100.0


# ------------------------------------------------------------------------------------------------------------------------
def test_whole_episode_production_noise_vs_oracle():
    """ParallelRunner.run at 64 envs x T = 90 with no noise hook (what bench.py times): K1 and K1c draw their own noise;
    the sampled envs must match the oracle fed the replayed Gumbel noise and uniforms (the assertions of
    test_whole_episode_device_runner_vs_oracle)."""
    _need_gpu()
    from iplan_b200.runners.synthetic_runner import build_system
    from oracle import philox as PX
    from tests.test_gpu_baseline_sizes import oracle_episode
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    B = 64
    sysm = build_system(n_envs=B, env="highway", hazard=0.01, seed=29)
    a = sysm.args
    A, N, T = a.n_agents, a.max_vehicle_num, a.episode_limit
    with torch.no_grad():
        for ag in sysm.mac.agents:
            ag.act.action_out.linear.weight.mul_(30.0)
    g0, c0 = sysm.prediction.calls, sysm.mac.calls
    batch, *_ = sysm.runner.run(test_mode=False)
    torch.cuda.synchronize()
    assert sysm.prediction.calls - g0 == T + 1 and sysm.mac.calls - c0 == T
    S = [0, 37, 63]
    seed_g, seed_c = sysm.prediction.seed, sysm.mac.seed
    rec = {"gumbel": [torch.as_tensor(PX.gat_step_gumbel(seed_g, g0 + k, A, B, N, envs=S)) for k in range(T + 1)],
           "uniforms": [torch.as_tensor(PX.controller_uniforms(seed_c, c0 + t, A, B)[:, S]) for t in range(T)]}
    worst, flips = oracle_episode(sysm, batch, S, rec)
    print(f"[episode, production noise, B={B} envs {S}] worst |cuda - oracle|: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + f"; sampled actions differing: {flips} of {T * A * len(S)}")
    assert flips <= 1
    assert all(v < TOL for v in worst.values()), worst


# ------------------------------------------------------------------------------------------------------------------------
def _pred_batch(args, B, T1, seed):
    from tools.check_beh_learn_tile import make_batch
    batch = make_batch(args, B, T1, seed)
    g = torch.Generator().manual_seed(seed + 1)
    A, N, L, D = args.n_agents, args.max_vehicle_num, args.latent_dim, args.attention_dim
    att = torch.rand(B, T1, A, N, D, generator=g) * 2 - 1
    beh = torch.softmax(torch.randn(B, T1, A, N, L, generator=g), -1)
    batch.update({"attention_latent": att.numpy(), "behavior_latent": beh.numpy()}, bs=slice(None), ts=slice(None))
    return batch


def test_prediction_learn_philox_vs_oracle():
    """Prediction_policy.learn at A = 5, P = 64, N = 55, pred_length = 5 with only select_idx given: the kernel draws its
    Gumbel noise and dropout.  Agent-nets 0 and 4 against the float64 oracle fed the replay (loss, every raw gradient
    tensor, post-step weights); then the replayed noise passed explicitly must give the Philox run's gradients within the
    run-to-run spread of the kernel's float atomics, measured by repeating the explicit call."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    args = make_args("highway", use_cuda=True, device="cuda", pred_batch_size=64, pred_length=5)
    A, N, P, pl, D = args.n_agents, args.max_vehicle_num, args.pred_batch_size, args.pred_length, args.attention_dim
    assert (A, N) == (5, 55)
    B, T1 = 4, 30
    batch = _pred_batch(args, B, T1, seed=31)
    avail_len = T1 - 1 - pl - 1
    rng = np.random.default_rng(32)
    sel = [rng.choice(B * avail_len, size=P, replace=False) for _ in range(A)]

    def fresh():
        torch.manual_seed(33)
        return Prediction_policy(args, None)

    pol = fresh()
    gat_before, dec_before = _params(pol.pred_GAT, torch.float64), _params(pol.pred_decoder, torch.float64)
    c0 = pol.calls
    pol.debug_learn = dict(select_idx=sel)
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    grads = {k: v.cpu() for k, v in pol.last_grads.items()}
    gum, keep = PX.pred_learn_noise(pol.seed, c0, A, P, N, pl, args.decoder_dropout)
    print(f"[pred learn] kept dropout fraction {keep.mean():.4f}")

    hist = batch["history"][:, :-1].cpu()
    att, beh = batch["attention_latent"][:, :-1].cpu(), batch["behavior_latent"][:, :-1].cpu()
    flag = batch["terminated"][:, :-1, :, 0].cpu()
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    offs = {"gat": pol.stack.named_offsets(), "dec": pol.dec_stack.named_offsets()}
    after = {a: {**{k: v.cpu() for k, v in pol.pred_GAT[a].state_dict().items()},
                 **{k: v.cpu() for k, v in pol.pred_decoder[a].state_dict().items()}} for a in (0, A - 1)}
    bad = []
    for a in (0, A - 1):
        refs = {}
        for dt in (torch.float64, torch.float32):
            gp = {k: v.to(dt).clone() for k, v in gat_before[a].items()}
            dp = {k: v.to(dt).clone() for k, v in dec_before[a].items()}
            ref, _ = O.prediction_learn_agent(gp, dp, hist[:, :, a].to(dt), att[:, :, a].to(dt), beh[:, :, a].to(dt), flag[:, :, a],
                                              torch.as_tensor(sel[a]), torch.as_tensor(gum[a]).to(dt),
                                              torch.as_tensor(keep[a]).permute(1, 0, 2, 3), oargs)
            refs[dt] = (ref, {**gp, **dp})
        (r64, w64), (r32, w32) = refs[torch.float64], refs[torch.float32]
        dl, sl = abs(float(losses[a]) - r64["loss"]) / abs(r64["loss"]), abs(r32["loss"] - r64["loss"]) / abs(r64["loss"])
        print(f"[pred learn a={a}] loss cuda {float(losses[a]):.7f} oracle64 {r64['loss']:.7f} rel {dl:.2e} (fp32 oracle {sl:.2e})")
        if dl > _bound(sl):
            bad.append((a, "loss"))
        mine = {}
        for kind in ("gat", "dec"):
            for name, (off, shape) in offs[kind].items():
                n = int(np.prod(shape)) if len(shape) else 1
                mine[name] = grads[kind][a, off:off + n].view(shape)
        bad += [(a, n) for n in _check_tensors("grad", mine, r64["grads"], r32["grads"])]
        bad += [(a, "w:" + n) for n in _check_tensors("weight", after[a], w64, w32, absolute=True)]

    # the same call with the replayed noise passed explicitly, twice: the atomics spread, and the Philox run inside it
    reps = []
    for _ in range(2):
        p2 = fresh()
        p2.debug_learn = dict(select_idx=sel, gumbel=torch.as_tensor(gum), keep=torch.as_tensor(keep))
        p2.learn(batch, t_env=0)
        torch.cuda.synchronize()
        reps.append({k: v.cpu() for k, v in p2.last_grads.items()})
    worst_spread, worst_gap = 0.0, 0.0
    for kind in ("gat", "dec"):
        for name, (off, shape) in offs[kind].items():
            n = int(np.prod(shape)) if len(shape) else 1
            for a in range(A):
                x1, x2, xp = (r[kind][a, off:off + n] for r in (reps[0], reps[1], grads))
                spread, gap = _rel(x2, x1), _rel(xp, x1)
                worst_spread, worst_gap = max(worst_spread, spread), max(worst_gap, gap)
                if gap > max(3 * spread, 1e-6):
                    bad.append((a, "philox vs explicit " + name, gap, spread))
    print(f"[pred learn] explicit replay vs Philox run: worst rel {worst_gap:.2e}; run-to-run spread of the explicit call "
          f"(float atomics): worst rel {worst_spread:.2e}")
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------------
def test_soft_behavior_learn_philox_vs_oracle():
    """Behavior_policy.learn (soft update, the default module) at A = 5, N = 55, B = 8, T = 90 — 440 chains per agent-net,
    six full 64-chain tiles and a ragged one, 79 overlapping window positions, agents terminating inside the episode — with
    the kernels' own dropout, replayed into the float64 oracle: losses, clipped gradients, post-step weights of every
    agent-net."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.nova.stable_behavior_policy import Behavior_policy
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    from tools.check_beh_learn_tile import make_batch
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    args = make_args("highway", use_cuda=True, device="cuda")
    A, N, W, B, T = args.n_agents, args.max_vehicle_num, args.max_history_len, 8, 90
    batch = make_batch(args, B, T + 1, seed=41)
    torch.manual_seed(42)
    pol = Behavior_policy(args, None)
    enc_before, dec_before = _params(pol.behavior_encoder, torch.float64), _params(pol.behavior_decoder, torch.float64)
    c0 = pol.learn_calls
    t0 = time.perf_counter()
    b_loss, _, _ = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    n_pos = T - 1 - W
    keep = PX.beh_learn_keep(pol.seed, c0, A, B, n_pos, N, W, args.decoder_dropout)
    hist = batch["history"][:, :-1].cpu()
    term = batch["terminated"][:, :-1, :, 0].cpu().double()
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    bad = []
    for a in range(A):
        k_o = torch.as_tensor(keep[a]).permute(1, 0, 2, 3, 4).reshape(n_pos, B * N, W, -1)
        refs = {}
        for dt in (torch.float64, torch.float32):
            ep = {k: v.to(dt).clone() for k, v in enc_before[a].items()}
            dp = {k: v.to(dt).clone() for k, v in dec_before[a].items()}
            ref, _ = O.behavior_learn_agent(ep, dp, hist[:, :, a].to(dt), term[:, :, a].to(dt), k_o, oargs)
            refs[dt] = (ref, {**{"enc:" + k: v for k, v in ep.items()}, **{"dec:" + k: v for k, v in dp.items()}})
        (r64, w64), (r32, w32) = refs[torch.float64], refs[torch.float32]
        dl = abs(float(b_loss[a]) - r64["behavior_loss"]) / abs(r64["behavior_loss"])
        sl = abs(r32["behavior_loss"] - r64["behavior_loss"]) / abs(r64["behavior_loss"])
        print(f"[soft beh learn a={a}] loss cuda {float(b_loss[a]):.7f} oracle64 {r64['behavior_loss']:.7f} rel {dl:.2e} (fp32 oracle {sl:.2e})")
        if dl > _bound(sl):
            bad.append((a, "loss"))
        mine = {}
        for kind, stack in (("enc", pol.stack), ("dec", pol.dec_stack)):
            flat = pol.last_grads[kind]
            raw = {name: flat[a, off:off + (int(np.prod(shape)) if len(shape) else 1)].view(shape).cpu()
                   for name, (off, shape) in stack.named_offsets().items()}
            total = torch.sqrt(sum((v.double() ** 2).sum() for v in raw.values()))
            coef = min(1.0, float(args.max_grad_norm) / (float(total) + 1e-6))
            mine.update({kind + ":" + n: v.double() * coef for n, v in raw.items()})
        bad += [(a, n) for n in _check_tensors("clipped grad", mine, r64["clipped"], r32["clipped"], floors=ENC_GRU_FLOOR)]
        after = {**{"enc:" + k: v.cpu() for k, v in pol.behavior_encoder[a].state_dict().items()},
                 **{"dec:" + k: v.cpu() for k, v in pol.behavior_decoder[a].state_dict().items()}}
        bad += [(a, "w:" + n) for n in _check_tensors("weight", after, w64, w32, absolute=True)]
    # the replayed mask passed explicitly, twice: the run-to-run spread of the kernels' float atomics, and the Philox run
    # inside it (the forward and the backward launches each draw the mask; any disagreement would show here)
    reps = []
    for _ in range(2):
        torch.manual_seed(42)
        p2 = Behavior_policy(args, None)
        p2.debug_keep = torch.as_tensor(keep)
        p2.learn(batch, t_env=0)
        torch.cuda.synchronize()
        reps.append({k: v.cpu() for k, v in p2.last_grads.items()})
    worst_spread, worst_gap = 0.0, 0.0
    for kind, stack in (("enc", pol.stack), ("dec", pol.dec_stack)):
        for name, (off, shape) in stack.named_offsets().items():
            n = int(np.prod(shape)) if len(shape) else 1
            for a in range(A):
                x1, x2 = reps[0][kind][a, off:off + n], reps[1][kind][a, off:off + n]
                xp = pol.last_grads[kind][a, off:off + n].cpu()
                spread, gap = _rel(x2, x1), _rel(xp, x1)
                worst_spread, worst_gap = max(worst_spread, spread), max(worst_gap, gap)
                if gap > max(3 * spread, 1e-6):
                    bad.append((a, "philox vs explicit " + kind + ":" + name, gap, spread))
    print(f"[soft beh learn] explicit replay vs Philox run: worst rel {worst_gap:.2e}; run-to-run spread of the explicit call "
          f"(float atomics): worst rel {worst_spread:.2e}; kept dropout fraction {keep.mean():.4f}; "
          f"test time {time.perf_counter() - t0:.1f} s")
    assert not bad, bad


def test_hard_behavior_learn_philox_vs_oracle():
    """The hard-update module's learn at the same shape (8 non-overlapping windows) with the kernels' own dropout,
    replayed into the float64 oracle through tools/check_beh_learn_hard.compare."""
    _need_gpu()
    import importlib
    chk = importlib.import_module("tools.check_beh_learn_hard")
    from iplan_b200.config import make_args
    from iplan_b200.nova.behavior_policy import Behavior_policy
    from oracle import philox as PX
    from tools.check_beh_learn_tile import make_batch
    args = make_args("highway", use_cuda=True, device="cuda", soft_update_enable=False)
    A, N, W, B, T = args.n_agents, args.max_vehicle_num, args.max_history_len, 8, 90
    batch = make_batch(args, B, T + 1, seed=51)
    torch.manual_seed(52)
    pol = Behavior_policy(args, None)
    enc_before, dec_before = _params(pol.behavior_encoder, torch.float64), _params(pol.behavior_decoder, torch.float64)
    pol.learn_calls = 3
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    n_pos = T // W - 1
    keep = PX.beh_learn_keep(pol.seed, 3, A, B, n_pos, N, W, args.decoder_dropout)
    keeps = [torch.as_tensor(keep[a]).permute(1, 0, 2, 3, 4).reshape(n_pos, B * N, W, -1) for a in range(A)]
    data = {"history": batch["history"].cpu().double(), "terminated": batch["terminated"].cpu()}
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    assert chk.compare(pol, data, keeps, oargs, enc_before, dec_before, losses, tag="hard, Philox dropout")


# ------------------------------------------------------------------------------------------------------------------------
def test_gat128_philox_equals_replayed_noise():
    """GAT128.forward drawing its own noise, then with the replay passed explicitly: the same output (to the accuracy of
    the kernel's fast logarithm, 1e-4)."""
    _need_gpu()
    from iplan_b200.nova.gat128 import GAT128, H, N
    from oracle import philox as PX
    A, items = 3, 64
    torch.manual_seed(61)
    net = GAT128(A, seed=5)
    with torch.no_grad():
        for k in ("hard_bi_GRU.weight_hh_l0", "hard_bi_GRU.weight_hh_l0_reverse", "hard_encoding.weight"):
            net.p[k].mul_(2.0)
    x = (torch.rand(A, items, N, H, device="cuda") * 2 - 1).contiguous()
    hp = torch.tanh(torch.randn(A, items, N, H, device="cuda")).contiguous()
    net.calls = 7
    out1 = net.forward(x, hp).clone()
    gum = torch.as_tensor(PX.gat128_gumbel(net.seed, 7, A, items)).cuda().contiguous()
    out2 = net.forward(x, hp, gumbel=gum)
    torch.cuda.synchronize()
    other = torch.as_tensor(PX.gat128_gumbel(net.seed, 8, A, items)).cuda().contiguous()
    out3 = net.forward(x, hp, gumbel=other)                  # the next counter's noise: a different output
    torch.cuda.synchronize()
    d, d_other = float((out1 - out2).abs().max()), float((out1 - out3).abs().max())
    print(f"[gat128 philox] max |Philox - replay| {d:.3e}; against the next counter's noise {d_other:.3e}")
    assert d < TOL and d_other > 100 * TOL
