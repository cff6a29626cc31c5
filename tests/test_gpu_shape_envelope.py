"""The kernels across the shapes their entry points accept, not only the two scenarios' shapes (MPE: 6 slots, obs_dim 4;
Hetero-Highway: 55 slots, obs_dim 5; latent 8, window 10, 5 actions).  Each case runs one kernel at an edge of its
envelope (slot counts around the 16-ego m-tiles and the 32-lane halves of K1, 1 to 8 actions, feature widths on both
staging paths of K1c, the largest slot count of each entry point, ragged 64-chain tiles of the behaviour learner) and
compares it with the float64 oracle (oracle/iplan_oracle.py, tools/beh_hard_oracle.py) fed the same noise: explicit
noise, plus one Philox case per kernel replayed with oracle/philox.py.

Tolerances as in the rest of the suite: 1e-4 absolute for rollout outputs; 1e-5 relative to each tensor's largest entry
for learner gradients (or 3x the float32 oracle's own distance from float64, where that is larger); hard-attention
gates only where the oracle's gate lies outside (0.01, 0.99).  Every case prints its worst error."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOL = 1e-4
GATE_TOL = 1e-3                 # a wrong draw or a wrong logit moves a well-conditioned gate by O(1)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _sd(stack, a, dtype=torch.float64):
    return {k: v.detach().cpu().to(dtype).clone() for k, v in stack.nets[a].state_dict().items()}


def _absmax(x, ref):
    return float((torch.as_tensor(x).double().cpu() - torch.as_tensor(ref).double().cpu()).abs().max()) if torch.as_tensor(ref).numel() else 0.0


def _nt():
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


# ---- K1: the GAT step ------------------------------------------------------------------------------------------------
K1_SLOTS = [2, 3, 4, 7, 16, 17, 32, 33, 48, 63, 64]
K1_DIMS = [(4, 8), (8, 8), (3, 2)]


def _k1_run(N, o, L, B=3, A=2, seed=0, philox=False):
    """K1 through the ABI at B envs x A agent-nets x N slots against O.gat_forward in float64: output, the per-edge logit
    differences the recurrence kernel hands to the attention kernel (the dl scratch) and the hard gates."""
    from iplan_b200 import _lib
    from iplan_b200.modules.flat import ParamStack
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    torch.manual_seed(seed)
    stack = ParamStack("gat", A, (o + L,))
    with torch.no_grad():                                   # a wider spread of hard-attention logits: both gate states occur
        for n in stack.nets:
            n.hard_encoding.weight.mul_(3.0)
    stack.to("cuda")
    g = torch.Generator().manual_seed(seed + 1)
    hist = torch.rand(A, B, N, o, generator=g) * 2 - 1
    hist[..., N // 2:, 0] = 0.0
    beh = torch.softmax(torch.randn(A, B, N, L, generator=g), -1) if L else torch.zeros(A, B, N, 0)
    att = torch.rand(A, B, N, 32, generator=g) * 2 - 1
    seed_k, counter = 1234 + N, 7
    if philox:
        gum = torch.as_tensor(PX.gat_step_gumbel(seed_k, counter, A, B, N)).float()
    else:
        gum = torch.stack([O.draw_gumbel(B * N * (N - 1), generator=g).view(B, N, N - 1, 2) for _ in range(A)])
    dev = lambda t: t.contiguous().cuda()
    h, b, hp = dev(hist), dev(beh) if L else torch.zeros(A, B, N, 1, device="cuda"), dev(att)
    out = torch.full((A, B, N, 32), float("nan"), device="cuda")
    hard = torch.full((A, B, N, N - 1), float("nan"), device="cuda")
    nsc = _lib.lib.iplan_gat_scratch_floats(B, A, N)
    scratch = torch.full((nsc,), float("nan"), device="cuda")
    rc = _lib.lib.iplan_gat_step(_lib.ptr(stack.flat), stack.stride(), _lib.view(h), _lib.view(b), _lib.view(hp),
                                 _lib.view(out), None if philox else _lib.ptr(dev(gum)), seed_k, counter, 0.01, _lib.ptr(hard),
                                 _lib.ptr(scratch), nsc, B, A, N, o, L, _lib.stream())
    _lib.check(rc, "gat_step")
    torch.cuda.synchronize()
    d_out, d_dl, d_gate, mid_frac = 0.0, 0.0, 0.0, 0.0
    dl = scratch.view(A, B, 2, N - 1, 64)[..., :N].sum(2).transpose(-1, -2).cpu().double()     # [A, B, N(ego), N-1(s)]
    for a in range(A):
        p = _sd(stack, a)
        x = torch.cat([hist[a], beh[a]], -1).double()
        ref, parts = O.gat_forward(p, x, att[a].reshape(B * N, 32).double(), gum[a].double(), return_parts=True)
        d_out = max(d_out, _absmax(out[a].reshape(B * N, 32), ref))
        lg = parts["logits"]
        want_dl = lg[..., 1] - lg[..., 0] - (p["hard_encoding.bias"][1] - p["hard_encoding.bias"][0])
        d_dl = max(d_dl, _absmax(dl[a], want_dl) / max(1.0, float(want_dl.abs().max())))
        rh = parts["hard"]
        ok = (rh <= 0.01) | (rh >= 0.99)
        mid_frac += float((~ok).double().mean()) / A
        if ok.any():
            d_gate = max(d_gate, float((hard[a].cpu().double() - rh).abs()[ok].max()))
    return d_out, d_dl, d_gate, mid_frac


@pytest.mark.parametrize("o,L", K1_DIMS)
@pytest.mark.parametrize("N", K1_SLOTS)
def test_k1_slot_counts_and_input_widths_vs_oracle64(N, o, L):
    _need_gpu()
    d_out, d_dl, d_gate, mid = _k1_run(N, o, L, B=3, seed=N * 10 + o)
    print(f"[K1 N={N} o={o} L={L} B=3] out {d_out:.2e}  dl {d_dl:.2e} (rel)  well-conditioned gates {d_gate:.2e} "
          f"(ill-conditioned fraction {mid:.3f})")
    assert d_out < TOL and d_dl < TOL and d_gate < GATE_TOL


@pytest.mark.parametrize("N", [2, 33, 64])
def test_k1_philox_noise_at_edge_slot_counts(N):
    """The kernel's own Gumbel noise (key (ego, j >> 2), words j & 3: keys up to 15 at N = 64) replayed into the oracle."""
    _need_gpu()
    d_out, d_dl, d_gate, mid = _k1_run(N, 5, 8, B=5, seed=N, philox=True)
    print(f"[K1 Philox N={N} B=5] out {d_out:.2e}  dl {d_dl:.2e}  well-conditioned gates {d_gate:.2e} (ill-conditioned {mid:.3f})")
    assert d_out < TOL and d_dl < TOL and d_gate < GATE_TOL


# ---- K1b: the behaviour-encoder step ---------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("o,W", [(1, 64), (4, 16), (7, 9), (5, 10)])
def test_k1b_window_and_latent_widths_vs_oracle64(o, W, L):
    """iplan_behavior_step on contiguous windows and iplan_behavior_step_ex on a time-strided store with a zero-padded
    front (win_pad > 0), at node counts (env x slot) of 21, 65 (ragged 16-node warps) and 128 (whole CTAs)."""
    _need_gpu()
    from iplan_b200 import _lib
    from iplan_b200.modules.flat import ParamStack
    from oracle import iplan_oracle as O
    A = 2
    torch.manual_seed(o * 100 + W + L)
    stack = ParamStack("beh", A, (o, L)).to("cuda")
    g = torch.Generator().manual_seed(o + W + L)
    worst = {}
    for (B, N), coef in (((3, 7), 0.1), ((5, 13), 1.0), ((2, 64), 0.1)):
        for strided in (False, True):
            pad = min(3, W - 1) if strided else 0
            T = W - pad + 2
            store = torch.rand(T, A, B, N, o, generator=g) * 2 - 1                 # [time][agent][env][slot][o]
            t0 = 1
            win = torch.zeros(A, B, N, W, o)
            win[:, :, :, pad:] = store[t0:t0 + W - pad].permute(1, 2, 3, 0, 4)
            hid = torch.rand(A, B, N, 32, generator=g) * 2 - 1
            prev = torch.softmax(torch.randn(A, B, N, L, generator=g), -1)
            hid_d, prev_d = hid.cuda(), prev.cuda()
            lat_d = torch.full((A, B, N, L), float("nan"), device="cuda")
            if strided:
                st = store.cuda()
                rc = _lib.lib.iplan_behavior_step_ex(_lib.ptr(stack.flat), stack.stride(), _lib.view(st[t0]), st.stride(0), pad,
                                                     _lib.view(hid_d), _lib.view(prev_d), _lib.view(lat_d), coef,
                                                     B, A, N, o, L, W, _lib.stream())
            else:
                wd = win.reshape(A, B, N, W * o).contiguous().cuda()
                rc = _lib.lib.iplan_behavior_step(_lib.ptr(stack.flat), stack.stride(), _lib.view(wd), _lib.view(hid_d),
                                                  _lib.view(prev_d), _lib.view(lat_d), coef, B, A, N, o, L, W, _lib.stream())
            _lib.check(rc, "behavior_step")
            torch.cuda.synchronize()
            dl, dh = 0.0, 0.0
            for a in range(A):
                h, z = O.behavior_encoder(_sd(stack, a), win[a].reshape(B * N, W, o).double(), hid[a].reshape(B * N, 32).double())
                new = (1 - coef) * prev[a].reshape(B * N, L).double() + coef * z
                dl = max(dl, _absmax(lat_d[a].reshape(B * N, L), new))
                dh = max(dh, _absmax(hid_d[a].reshape(B * N, 32), h))
            worst[(B * N, coef, "ex" if strided else "plain")] = (dl, dh)
    print(f"[K1b o={o} W={W} L={L}] worst (latent, hidden): " + "  ".join(f"{k}: {v[0]:.1e} {v[1]:.1e}" for k, v in worst.items()))
    assert all(max(v) < TOL for v in worst.values()), worst


# ---- K1c: the controller step ----------------------------------------------------------------------------------------
CTRL_FEATS = [37, 2485, 2561, 2800]          # 2561: past the vector staging path (K16 > 2560); 2800: IPLAN_CTRL_MAX_FEAT


def _masks(B, nA, g):
    """uint8 [B, nA] availability: all, the last action masked, all but one masked (cycling the one), random."""
    av = torch.ones(B, nA, dtype=torch.uint8)
    for b in range(B):
        k = b % 4
        if k == 1 and nA > 1:
            av[b, -1] = 0
        elif k == 2:
            av[b] = 0
            av[b, b % nA] = 1
        elif k == 3 and nA > 1:
            av[b] = (torch.rand(nA, generator=g) < 0.6).to(torch.uint8)
            av[b, (b // 4) % nA] = 1
    return av


def _ctrl_case(F, nA, B, greedy, pitch=None, philox=False, seed=0):
    from iplan_b200 import _lib
    from iplan_b200.modules.flat import ParamStack
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    A = 2
    torch.manual_seed(seed)
    ast, cst = ParamStack("actor", A, (F, nA)), ParamStack("critic", A, (F,))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n in ast.nets:
            n.act.action_out.linear.weight.mul_(30.0)
        for n in ast.nets + cst.nets:                                           # feature_norm weight | bias away from (1, 0)
            n.base.feature_norm.weight.copy_(torch.rand(F, generator=g) + 0.5)
            n.base.feature_norm.bias.copy_(torch.rand(F, generator=g) + 0.5)
    ast.to("cuda"), cst.to("cuda")
    pitch = pitch or F
    store = torch.zeros(A, B, pitch)
    x = torch.rand(A, B, F, generator=g) * 2 - 1
    store[:, :, :F] = x
    ra, rc_ = torch.rand(A, B, 64, generator=g) * 2 - 1, torch.rand(A, B, 64, generator=g) * 2 - 1
    av = torch.stack([_masks(B, nA, g) for _ in range(A)])                       # [A, B, nA]
    seed_k, counter = 77, 5
    uni = torch.as_tensor(PX.controller_uniforms(seed_k, counter, A, B)).float() if philox else torch.rand(A, B, generator=g)
    feat = store.cuda()
    na, nc = torch.empty(A, B, 64, device="cuda"), torch.empty(A, B, 64, device="cuda")
    act = torch.full((A, B), -1, dtype=torch.int32, device="cuda")
    lp, val = torch.empty(A, B, device="cuda"), torch.empty(A, B, device="cuda")
    logits = torch.empty(A, B, nA, device="cuda")
    ra_d, rc_d, av_d, uni_d = ra.cuda(), rc_.cuda(), av.cuda(), uni.contiguous().cuda()
    rc = _lib.lib.iplan_controller_step(_lib.ptr(ast.flat), ast.stride(), _lib.ptr(cst.flat), cst.stride(),
                                        _lib.ptr(feat), feat.stride(0), feat.stride(1), _lib.ptr(ra_d), _lib.ptr(rc_d),
                                        _lib.ptr(na), _lib.ptr(nc), 64 * B, 64, 64 * B, 64, _lib.ptr(av_d),
                                        None if philox else _lib.ptr(uni_d), seed_k, counter, 1 if greedy else 0,
                                        _lib.ptr(act), _lib.ptr(lp), _lib.ptr(val), _lib.ptr(logits), None, None,
                                        B, A, F, nA, _lib.stream())
    _lib.check(rc, "controller_step")
    torch.cuda.synchronize()
    ap = [_sd(ast, a) for a in range(A)]
    cp = [_sd(cst, a) for a in range(A)]
    t = lambda z: z.permute(1, 0, *range(2, z.dim())).double()
    ref = O.select_actions(ap, cp, t(x), t(av).long(), t(ra), t(rc_), test_mode=greedy, uniforms=t(uni))
    lg, keep = t(logits.cpu()), ref["logits"] > -1e9
    act_c = t(act.cpu()).long()
    same = act_c == ref["actions"]
    avail_ok = bool(torch.gather(t(av), 2, act_c.clamp(0, nA - 1).unsqueeze(-1)).all()) and bool((act_c >= 0).all())
    err = dict(logits=_absmax(lg[keep], ref["logits"][keep]), value=_absmax(t(val.cpu()), ref["values"]),
               rnn_a=_absmax(t(na.cpu()), ref["rnn_a"]), rnn_c=_absmax(t(nc.cpu()), ref["rnn_c"]),
               logp=_absmax(t(lp.cpu())[same], ref["logp"][same]) if same.any() else 0.0)
    return err, int((~same).sum()), avail_ok


@pytest.mark.parametrize("F", CTRL_FEATS)
@pytest.mark.parametrize("nA", [1, 2, 6, 8])
def test_k1c_action_counts_envs_and_feature_widths_vs_oracle64(nA, F):
    """Sampled and greedy, at n_envs around CTRL_ROWS = 18 rows per CTA; masks with the last action off and with all but
    one off.  A sampled action may differ only where its uniform lies within float32 noise of a cdf edge: at most one per
    case, and every chosen action is available."""
    _need_gpu()
    bad, report = [], []
    for B in (1, 17, 18, 19, 37):
        for greedy in (False, True):
            err, flips, avail_ok = _ctrl_case(F, nA, B, greedy, seed=F + 10 * nA + B)
            w = max(err.values())
            report.append(f"B={B}{'g' if greedy else 's'} {w:.1e}/{flips}")
            if w >= TOL or flips > 1 or not avail_ok:
                bad.append((B, greedy, err, flips, avail_ok))
    print(f"[K1c nA={nA} F={F}] worst error / differing actions: " + "  ".join(report))
    assert not bad, bad


def test_k1c_scalar_staging_path_for_an_unaligned_row_pitch():
    """Rows 2487 floats apart (not a multiple of 4): K1c stages them on its scalar path; the same rows at pitch 2488 take the
    vector path.  Both against the oracle, with 8 actions and Philox sampling replayed."""
    _need_gpu()
    for pitch in (2487, 2488):
        err, flips, avail_ok = _ctrl_case(2485, 8, 37, False, pitch=pitch, philox=True, seed=pitch)
        print(f"[K1c F=2485 pitch {pitch}, Philox] {err} differing actions {flips}")
        assert max(err.values()) < TOL and flips <= 1 and avail_ok


# ---- IPPO learner at 6 and 8 actions -----------------------------------------------------------------------------------
def masked_mpe_learner_case(nA, B, T, seed, **overrides):
    """Learner inputs at the 7-slot MPE width (3 agents, 3 landmarks, 1 random agent: feat_dim 308 + nA + 3, not a
    multiple of 32) with nA actions: B episodes of T steps, random availability masks (the action taken is always
    available), terminations of 3 % per step, a x30 policy head.  Returns (args, data, actors, critics, feat_dim)."""
    from iplan_b200.config import controller_input_dim, make_args
    from iplan_b200.modules.flat import ParamStack
    args = make_args("MPE", num_random_agents=1, n_actions=nA, episode_limit=T, batch_size_run=B, buffer_size=B,
                     batch_size=B - 1, use_cuda=True, device="cuda", **overrides)
    A, N, o, L, D, R = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim, args.rnn_hidden_dim
    assert N == 7
    F = controller_input_dim(args)
    assert F == 308 + nA + A and F % 32 != 0
    rng = np.random.default_rng(seed)
    hist = rng.uniform(-1, 1, size=(B, T + 1, A, N, o)).astype(np.float32)
    acts = rng.integers(0, nA, size=(B, T + 1, A, 1))
    avail = (rng.uniform(size=(B, T + 1, A, nA)) < 0.5).astype(np.int64)
    np.put_along_axis(avail, acts, 1, axis=-1)                       # the action taken is always available
    term = (np.cumsum(rng.uniform(size=(B, T + 1, A, 1)) < 0.03, axis=1) > 0).astype(np.uint8)
    data = dict(history=hist, attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
                behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
                rnn_states_actors=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                rnn_states_critics=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                actions=acts, avail_actions=avail, reward=(rng.normal(size=(B, T + 1, A, 1)) * 2).astype(np.float32),
                terminated=term)
    torch.manual_seed(seed)
    a0, c0 = ParamStack("actor", A, (F, nA)), ParamStack("critic", A, (F,))
    with torch.no_grad():
        for n in a0.nets:
            n.act.action_out.linear.weight.mul_(30.0)
    actors = [{k: v.clone() for k, v in n.state_dict().items()} for n in a0.nets]
    critics = [{k: v.clone() for k, v in n.state_dict().items()} for n in c0.nets]
    return args, data, actors, critics, F


@pytest.mark.parametrize("nA", [6, 8])
def test_learner_six_and_eight_actions_vs_oracle(nA):
    """IPPOLearner.train at the 7-slot MPE width (3 agents, 3 landmarks, 1 random agent: feat_dim 308 + nA + 3, not a
    multiple of 32) with nA actions, many rows masking actions other than the one taken: first-epoch gradients of agent 1
    against O.train_agent, post-update weights with the bounds of test_learner_vs_oracle_baseline_shape."""
    _need_gpu()
    import importlib.util
    spec = importlib.util.spec_from_file_location("test_gpu_learner", os.path.join(ROOT, "tests", "test_gpu_learner.py"))
    tgl = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tgl)
    from oracle import iplan_oracle as O
    _nt()
    B, T = 12, 20
    args, data, actors, critics, F = masked_mpe_learner_case(nA, B, T, seed=nA)
    batch, mac, learner, _ = tgl.build(args, data, actors, critics)
    learner.keep_pre = True
    learner.insert_episode_batch(batch)
    learner.train(0)
    torch.cuda.synchronize()
    ag = 1
    dt = {k: torch.as_tensor(v) for k, v in data.items()}
    onehot = torch.nn.functional.one_hot(dt["actions"].squeeze(-1), nA).float()
    ob = dict(history=dt["history"][:, :, ag], attention_latent=dt["attention_latent"][:, :, ag],
              behavior_latent=dt["behavior_latent"][:, :, ag], actions=dt["actions"][:, :, ag],
              actions_onehot=onehot[:, :, ag], available_actions=dt["avail_actions"][:, :, ag],
              reward=dt["reward"][:, :, ag], terminated_masks=(1 - dt["terminated"][:, :, ag].float()),
              rnn_states_actor=dt["rnn_states_actors"][:, :, ag], rnn_states_critic=dt["rnn_states_critics"][:, :, ag])
    perms = [torch.randperm(args.batch_size * T, generator=torch.Generator().manual_seed(100 + e)) for e in range(args.ppo_epoch)]
    dbl = lambda d: {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}
    ap, cp = {k: v.clone() for k, v in actors[ag].items()}, {k: v.clone() for k, v in critics[ag].items()}
    ap64, cp64 = dbl({k: v.clone() for k, v in actors[ag].items()}), dbl({k: v.clone() for k, v in critics[ag].items()})
    stats64, pre64, _, _ = O.train_agent(ap64, cp64, dbl(ob), ag, SimpleNamespace(**vars(args)), perms=perms)
    O.train_agent(ap, cp, ob, ag, SimpleNamespace(**vars(args)), perms=perms)
    mine = learner.last_pre
    dpre = {k: _absmax(mine[k][ag], pre64[k]) for k in ("values_all", "returns", "advantages", "old_logp")}
    offs = {"actor": mac.actor_stack.named_offsets(), "critic": mac.critic_stack.named_offsets()}
    worst_grad = 0.0
    for kind, key in (("actor", "grads_actor"), ("critic", "grads_critic")):
        for name, gref in stats64[0][key].items():
            off, shape = offs[kind][name]
            gm = learner.first_grads[kind][ag, off:off + gref.numel()].view(gref.shape).cpu().double()
            worst_grad = max(worst_grad, float((gm - gref).abs().max() / (gref.abs().max() + 1e-12)))
    worst_w, n_off, n_all, sq_dev, sq_moved, ref_w = 0.0, 0, 0, 0.0, 0.0, 0.0
    for nets, ref32, ref64, init in ((mac.agents, ap, ap64, actors[ag]), (mac.critics, cp, cp64, critics[ag])):
        sd = nets[ag].state_dict()
        for k, v in ref64.items():
            d = (sd[k].detach().cpu().double() - v.detach()).abs()
            mv = v.detach() - init[k].double()
            worst_w = max(worst_w, float(d.max()) if d.numel() else 0.0)
            ref_w = max(ref_w, _absmax(ref32[k].detach(), v.detach()) if d.numel() else 0.0)
            n_off += int((d > 5e-5).sum())
            n_all += d.numel()
            sq_dev += float((d * d).sum()); sq_moved += float((mv * mv).sum())
    rms_dev, rms_moved = (sq_dev / n_all) ** 0.5, (sq_moved / n_all) ** 0.5
    print(f"[learner nA={nA} F={F}, agent {ag}] pre {dpre}; first-epoch grad rel {worst_grad:.2e}; post-update weights vs fp64: "
          f"worst {worst_w:.2e} (fp32 oracle {ref_w:.2e}), rms {rms_dev:.2e} of movement {rms_moved:.2e}, {n_off}/{n_all} > 5e-5")
    assert all(v < 2e-4 for v in dpre.values()), dpre
    assert worst_grad < 1e-5
    assert worst_w < args.lr and rms_dev < 0.02 * rms_moved and n_off <= 0.005 * n_all


# ---- Prediction_policy.learn -------------------------------------------------------------------------------------------
def _learn_batch(args, B, T1, seed):
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from tools.check_pred_learn import scheme_for
    A, N, o, L, D = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim
    g = torch.Generator().manual_seed(seed)
    scheme, groups, pre = scheme_for(args)
    batch = EpisodeBatch(scheme, groups, B, T1, preprocess=pre, device="cuda")
    hist = torch.rand(B, T1, A, N, o, generator=g) * 2 - 1
    hist[..., 0] = 1.0
    hist[:, :, :, (N + 1) // 2:][torch.rand(B, T1, A, 1, generator=g).expand(-1, -1, -1, N - (N + 1) // 2) < 0.3] = 0.0
    # every (env, agent) terminates at a step in [1, T1 / 2]: both learners weigh the rows from there on (the reference's
    # masks), so every case has a loss
    stop = torch.randint(1, max(2, T1 // 2 + 1), (B, 1, A), generator=g)
    term = (torch.arange(T1).view(1, T1, 1) >= stop).to(torch.uint8).unsqueeze(-1)
    upd = {"history": hist.numpy(), "terminated": term.numpy()}
    if "attention_latent" in scheme:
        upd["attention_latent"] = (torch.rand(B, T1, A, N, D, generator=g) * 2 - 1).numpy()
        upd["behavior_latent"] = torch.softmax(torch.randn(B, T1, A, N, L, generator=g), -1).numpy()
    batch.update(upd, bs=slice(None), ts=slice(None))
    return batch


def _check_tensors(tag, mine, o64, o32, absolute=False, floors=None):
    from tests.test_gpu_noise_streams import _check_tensors as chk
    return chk(tag, mine, o64, o32, absolute=absolute, floors=floors)


def _loss_rel(got, r64, r32):
    """(relative error of the loss, its bound: 1e-5 or 3x the float32 oracle's own error)"""
    dl, sl = abs(float(got) - r64) / abs(r64), abs(float(r32) - r64) / abs(r64)
    return dl, max(1e-5, 3 * sl)


@pytest.mark.parametrize("pl", [1, 5])
@pytest.mark.parametrize("N", [2, 7, 17, 57])
def test_prediction_learn_slot_counts_vs_oracle64(N, pl):
    """Prediction_policy.learn at obs_dim + latent_dim = 16 (8 + 8), N up to IPLAN_PRED_LEARN_MAX_SLOTS = 57, explicit
    Gumbel noise and dropout (Philox, replayed, at N = 17): the loss and every raw gradient tensor of both agent-nets."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    _nt()
    A, P, B, T1 = 2, 6, 3, 14
    philox = N == 17
    args = make_args("highway", n_agents=A, n_other_vehicles=N - A, obs_shape_single=8, latent_dim=8, pred_batch_size=P,
                     pred_length=pl, use_cuda=True, device="cuda")
    assert args.max_vehicle_num == N
    batch = _learn_batch(args, B, T1, seed=N + pl)
    avail_len = T1 - 1 - pl - 1
    rng = np.random.default_rng(N)
    sel = [rng.choice(B * avail_len, size=P, replace=False) for _ in range(A)]
    torch.manual_seed(N)
    pol = Prediction_policy(args, None)
    gat0 = [_sd(pol.stack, a) for a in range(A)]
    dec0 = [_sd(pol.dec_stack, a) for a in range(A)]
    if philox:
        gum, keep = PX.pred_learn_noise(pol.seed, pol.calls, A, P, N, pl, args.decoder_dropout)
        pol.debug_learn = dict(select_idx=sel)
    else:
        g = torch.Generator().manual_seed(N * 7 + pl)
        gum = -torch.log(torch.empty(A, P, N, N - 1, 2).exponential_(generator=g))
        keep = (torch.rand(A, P, pl, N, 32, generator=g) >= args.decoder_dropout).to(torch.uint8)
        pol.debug_learn = dict(select_idx=sel, gumbel=gum, keep=keep)
    losses = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    hist = batch["history"][:, :-1].cpu()
    att, beh = batch["attention_latent"][:, :-1].cpu(), batch["behavior_latent"][:, :-1].cpu()
    flag = batch["terminated"][:, :-1, :, 0].cpu()
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    offs = {"gat": pol.stack.named_offsets(), "dec": pol.dec_stack.named_offsets()}
    bad = []
    for a in range(A):
        refs = {}
        for dt in (torch.float64, torch.float32):
            gp = {k: v.to(dt).clone() for k, v in gat0[a].items()}
            dp = {k: v.to(dt).clone() for k, v in dec0[a].items()}
            refs[dt], _ = O.prediction_learn_agent(gp, dp, hist[:, :, a].to(dt), att[:, :, a].to(dt), beh[:, :, a].to(dt),
                                                   flag[:, :, a], torch.as_tensor(sel[a]), torch.as_tensor(gum[a]).to(dt),
                                                   torch.as_tensor(keep[a]).permute(1, 0, 2, 3), oargs)
        r64, r32 = refs[torch.float64], refs[torch.float32]
        assert r64["loss"] != 0.0, "no unmasked sample: the case tests nothing"
        dl, bound = _loss_rel(losses[a], r64["loss"], r32["loss"])
        print(f"[pred learn N={N} pl={pl}{' Philox' if philox else ''} a={a}] loss rel {dl:.2e}")
        if dl > bound:
            bad.append((a, "loss", dl))
        mine = {}
        for kind in ("gat", "dec"):
            for name, (off, shape) in offs[kind].items():
                n = int(np.prod(shape)) if len(shape) else 1
                mine[name] = pol.last_grads[kind][a, off:off + n].view(shape).cpu()
        # With few edges (N = 2: one per ego) every hard-attention gate can sit deep in saturation (tau = 0.01): the hard
        # path's gradients are then 1e-20 and smaller, below float32 resolution of the update (the kernel's fast exp
        # flushes them to zero).  Tensors under 1e-6 of the agent-net's largest gradient entry are held to an absolute
        # bound at that scale instead.
        top = max(float(v.abs().max()) for v in r64["grads"].values())
        tiny = [n for n, v in r64["grads"].items() if float(v.abs().max()) < 1e-6 * top]
        for n in tiny:
            d = _absmax(mine[n], r64["grads"][n])
            print(f"    grad {n:34s} below resolution: oracle max {float(r64['grads'][n].abs().max()):.1e}, |cuda - oracle| {d:.1e} "
                  f"(bound {1e-5 * top:.1e})")
            if d > 1e-5 * top:
                bad.append((a, n, d))
        keep_n = [n for n in r64["grads"] if n not in tiny]
        bad += [(a, n) for n in _check_tensors("grad", {n: mine[n] for n in keep_n}, {n: r64["grads"][n] for n in keep_n},
                                              {n: r32["grads"][n] for n in keep_n})]
    assert not bad, bad


# ---- Behavior_policy.learn: soft and hard window geometry ----------------------------------------------------------
BEH_CHAINS = {1: (1, 1), 63: (9, 7), 64: (8, 8), 65: (5, 13), 129: (3, 43)}    # B * N chains per agent-net: (B, N)


@pytest.mark.parametrize("chains", sorted(BEH_CHAINS))
@pytest.mark.parametrize("W", [1, 2, 10])
@pytest.mark.parametrize("o,L", [(1, 2), (7, 8)])
@pytest.mark.parametrize("hard", [False, True])
def test_behavior_learn_windows_vs_oracle64(hard, o, L, W, chains):
    """The soft module's learn (overlapping windows, geometry (1, 1 - W)) and the hard module's (non-overlapping, (W, 0))
    at B * N chains per agent-net around the 64-chain tile, explicit dropout (Philox, replayed, at 65 chains): losses,
    clipped gradients and post-step weights of both agent-nets against the float64 oracle."""
    _need_gpu()
    from iplan_b200.config import make_args
    from oracle import iplan_oracle as O
    from oracle import philox as PX
    from tests.test_gpu_noise_streams import ENC_GRU_FLOOR
    from tools.beh_hard_oracle import behavior_learn_hard_agent
    _nt()
    B, N = BEH_CHAINS[chains]
    A = 1 if N == 1 else 2
    philox = chains == 65
    args = make_args("highway", n_agents=A, n_other_vehicles=N - A, obs_shape_single=o, latent_dim=L, max_history_len=W,
                     soft_update_enable=not hard, use_cuda=True, device="cuda")
    if hard:
        from iplan_b200.nova.behavior_policy import Behavior_policy
        T = 4 * W
        n_pos = T // W - 1
    else:
        from iplan_b200.nova.stable_behavior_policy import Behavior_policy
        T = W + 4
        n_pos = T - 1 - W
    batch = _learn_batch(args, B, T + 1, seed=chains + W + o)
    torch.manual_seed(chains + 3 * W)
    pol = Behavior_policy(args, None)
    enc0 = [_sd(pol.stack, a) for a in range(A)]
    dec0 = [_sd(pol.dec_stack, a) for a in range(A)]
    if philox:
        keep = torch.as_tensor(PX.beh_learn_keep(pol.seed, pol.learn_calls, A, B, n_pos, N, W, args.decoder_dropout))
    else:
        g = torch.Generator().manual_seed(chains * 31 + W)
        keep = (torch.rand(A, B, n_pos, N, W, 64, generator=g) >= args.decoder_dropout).to(torch.uint8)
        pol.debug_keep = keep
    out = pol.learn(batch, t_env=0)
    torch.cuda.synchronize()
    losses = out if hard else out[0]
    hist = batch["history"][:, :-1].cpu()
    term = batch["terminated"][:, :-1, :, 0].cpu().double()
    oargs = SimpleNamespace(**{k: v for k, v in vars(args).items() if isinstance(v, (int, float, str, bool))})
    bad = []
    for a in range(A):
        k_o = keep[a].permute(1, 0, 2, 3, 4).reshape(n_pos, B * N, W, -1)
        refs = {}
        for dt in (torch.float64, torch.float32):
            ep = {k: v.to(dt).clone() for k, v in enc0[a].items()}
            dp = {k: v.to(dt).clone() for k, v in dec0[a].items()}
            if hard:
                ref, _ = behavior_learn_hard_agent(ep, dp, hist[:, :, a].to(dt), term[:, :, a].to(dt), k_o, oargs)
            else:
                ref, _ = O.behavior_learn_agent(ep, dp, hist[:, :, a].to(dt), term[:, :, a].to(dt), k_o, oargs)
            refs[dt] = (ref, {**{"enc:" + k: v for k, v in ep.items()}, **{"dec:" + k: v for k, v in dp.items()}})
        (r64, w64), (r32, w32) = refs[torch.float64], refs[torch.float32]
        dl, bound = _loss_rel(losses[a], r64["behavior_loss"], r32["behavior_loss"])
        print(f"[beh learn {'hard' if hard else 'soft'} o={o} L={L} W={W} chains={chains}{' Philox' if philox else ''} a={a}] "
              f"loss rel {dl:.2e}")
        if dl > bound:
            bad.append((a, "loss", dl))
        mine = {}
        for kind, stack in (("enc", pol.stack), ("dec", pol.dec_stack)):
            flat = pol.last_grads[kind]
            raw = {name: flat[a, off:off + (int(np.prod(shape)) if len(shape) else 1)].view(shape).cpu()
                   for name, (off, shape) in stack.named_offsets().items()}
            total = torch.sqrt(sum((v.double() ** 2).sum() for v in raw.values()))
            coef = min(1.0, float(args.max_grad_norm) / (float(total) + 1e-6))
            mine.update({kind + ":" + n: v.double() * coef for n, v in raw.items()})
        bad += [(a, n) for n in _check_tensors("clipped grad", mine, r64["clipped"], r32["clipped"], floors=None if hard else ENC_GRU_FLOOR)]
        after = {**{"enc:" + k: v.cpu() for k, v in pol.behavior_encoder[a].state_dict().items()},
                 **{"dec:" + k: v.cpu() for k, v in pol.behavior_decoder[a].state_dict().items()}}
        bad += [(a, "w:" + n) for n in _check_tensors("weight", after, w64, w32, absolute=True)]
    assert not bad, bad


# ---- whole episodes ----------------------------------------------------------------------------------------------------
def _episode(sysm, S, seed):
    from tests.test_gpu_baseline_sizes import oracle_episode
    a = sysm.args
    A, N, T, B = a.n_agents, a.max_vehicle_num, a.episode_limit, a.batch_size_run
    with torch.no_grad():
        for ag in sysm.mac.agents:
            ag.act.action_out.linear.weight.mul_(30.0)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    rec = {"gumbel": [], "uniforms": []}

    def noise(kind, idx):
        if kind == "gumbel":
            g = -torch.log(torch.empty(A, B, N, N - 1, 2, device="cuda").exponential_(generator=gen))
            rec["gumbel"].append(g[:, S].cpu())
            return g
        u = torch.rand(A, B, device="cuda", generator=gen)
        rec["uniforms"].append(u[:, S].cpu())
        return u

    sysm.runner.noise_hook = noise
    batch, *_ = sysm.runner.run(test_mode=False)
    torch.cuda.synchronize()
    assert len(rec["gumbel"]) == T + 1 and len(rec["uniforms"]) == T
    return oracle_episode(sysm, batch, S, rec)


def test_episode_mpe_with_a_random_agent():
    """simple_spread_Hetero with one random agent (3 agents + 3 landmarks + 1 = 7 slots), a short episode through the
    device runner against the oracle stepping the same episode."""
    _need_gpu()
    from iplan_b200.runners.synthetic_runner import build_system
    _nt()
    sysm = build_system(n_envs=9, env="MPE", num_random_agents=1, episode_limit=12, seed=71)
    assert sysm.args.max_vehicle_num == 7
    S = [0, 4, 8]
    worst, flips = _episode(sysm, S, seed=72)
    print(f"[episode MPE N=7] worst: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()) + f"; flips {flips}")
    assert flips <= 1 and all(v < TOL for v in worst.values()), worst


def test_episode_highway_at_the_largest_slot_count_the_rollout_accepts():
    """Hetero-Highway widths at n_other_vehicles = 57: N = 62 slots, controller input 2800 floats (IPLAN_CTRL_MAX_FEAT,
    the scalar staging path of K1c).  One more slot is rejected (tests/test_shape_envelope_cpu.py)."""
    _need_gpu()
    from iplan_b200.config import controller_input_dim
    from iplan_b200.runners.synthetic_runner import build_system
    _nt()
    sysm = build_system(n_envs=3, env="highway", n_other_vehicles=57, episode_limit=8, hazard=0.05, seed=81)
    assert sysm.args.max_vehicle_num == 62 and controller_input_dim(sysm.args) == 2800
    S = [0, 2]
    worst, flips = _episode(sysm, S, seed=82)
    print(f"[episode Highway N=62] worst: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()) + f"; flips {flips}")
    assert flips <= 1 and all(v < TOL for v in worst.values()), worst
