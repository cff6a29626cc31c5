"""Parity of the CUDA rollout kernels (K1 GAT, K1b behaviour encoder, K1c controller),
called through the reference-facing classes / the C ABI, against
 (1) the committed golden outputs of the reference's own modules, and
 (2) the CPU oracle on seeded inputs at the Highway shape.
Tolerance: 1e-4 (north_star: logits / values within 1e-4 rel fp32)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def maxdiff(a, b):
    a = torch.as_tensor(np.asarray(a.detach().cpu()) if torch.is_tensor(a) else np.asarray(a)).double()
    b = torch.as_tensor(np.asarray(b.detach().cpu()) if torch.is_tensor(b) else np.asarray(b)).double()
    return float((a - b).abs().max())


def args_from(d, **over):
    from iplan_b200.config import make_args
    env = d.get("env", "highway")
    a = make_args(env)
    for k, v in d.items():
        setattr(a, k, v)
    a.use_cuda, a.device = True, "cuda"
    for k, v in over.items():
        setattr(a, k, v)
    return a


def make_scheme(args):
    from iplan_b200.components.transforms import OneHot
    scheme = {
        "state": {"vshape": args.state_shape},
        "obs": {"vshape": args.obs_shape, "group": "agents"},
        "actions": {"vshape": (1,), "group": "agents", "dtype": torch.long},
        "rnn_states_actors": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "rnn_states_critics": {"vshape": (args.rnn_hidden_dim,), "group": "agents"},
        "history": {"vshape": (args.max_vehicle_num, args.obs_shape_single,), "group": "agents"},
        "behavior_latent": {"vshape": (args.max_vehicle_num, args.latent_dim,), "group": "agents"},
        "attention_latent": {"vshape": (args.max_vehicle_num, args.attention_dim,), "group": "agents"},
        "avail_actions": {"vshape": (args.n_actions,), "group": "agents", "dtype": torch.int},
        "reward": {"vshape": (1,), "group": "agents"},
        "speed": {"vshape": (1,), "group": "agents"},
        "terminated": {"vshape": (1,), "group": "agents", "dtype": torch.uint8},
    }
    return scheme, {"agents": args.n_agents}, {"actions": ("actions_onehot", [OneHot(out_dim=args.n_actions)])}


# ------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_gat_kernel_vs_reference_golden(golden_dir, case):
    """GAT_Net.forward golden (one agent-net) through the raw C ABI."""
    _need_gpu()
    from iplan_b200 import _lib
    from iplan_b200.modules.flat import ParamStack
    g = load(golden_dir, "gat_net.pt")[case]
    d = g["dims"]
    B, N, o, L, D = d["B"], d["N"], d["o"], d["L"], d["D"]
    stack = ParamStack("gat", 1, (o + L,), device="cuda")
    stack.nets[0].load_state_dict(g["params"])
    obs = g["obs"].cuda()
    hist = obs[..., :o].contiguous().view(1, B, N, o)
    beh = obs[..., o:].contiguous().view(1, B, N, L)
    hprev = g["h_prev"].cuda().view(1, B, N, D)
    out = torch.zeros(1, B, N, D, device="cuda")
    hard = torch.zeros(1, B, N, N - 1, device="cuda")
    gum = g["gumbel"].cuda().view(1, B, N, N - 1, 2).contiguous()
    scratch = torch.empty(_lib.lib.iplan_gat_scratch_floats(B, 1, N), device="cuda")
    rc = _lib.lib.iplan_gat_step(_lib.ptr(stack.flat), stack.stride(), _lib.view(hist), _lib.view(beh),
                                 _lib.view(hprev), _lib.view(out), _lib.ptr(gum), 1, 0, 0.01, _lib.ptr(hard),
                                 _lib.ptr(scratch), scratch.numel(), B, 1, N, o, L, _lib.stream())
    _lib.check(rc, "gat_step")
    torch.cuda.synchronize()
    from oracle import iplan_oracle as O
    _, parts = O.gat_forward(g["params"], g["obs"], g["h_prev"], g["gumbel"], return_parts=True)
    dh = maxdiff(hard.view(B, N, N - 1), parts["hard"])
    dout = maxdiff(out.view(B * N, D), g["out"])
    print(f"[gat {case}] max|hard diff|={dh:.3e} max|out diff|={dout:.3e}")
    assert dout < TOL, (dh, dout)


def test_rollout_modules_vs_reference_golden(golden_dir):
    """Prediction_policy.GAT_latent_update -> Behavior_policy.latent_update ->
    EpisodeBatch.update -> DcntrlMAC.select_actions_ippo, three consecutive steps, both
    golden cases, through the reference-facing numpy API."""
    _need_gpu()
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from iplan_b200.nova.stable_behavior_policy import Behavior_policy
    for case in ("mpe", "highway"):
        g = load(golden_dir, "rollout_modules.pt")[case]
        args = args_from(g["args"])
        A = args.n_agents
        B = args.batch_size_run
        T = args.episode_limit
        pred, beh = Prediction_policy(args, None), Behavior_policy(args, None)
        scheme, groups, pre = make_scheme(args)
        batch = EpisodeBatch(scheme, groups, B, T + 1, preprocess=pre, device="cuda")
        mac = DcntrlMAC(batch.scheme, groups, args)
        for i in range(A):
            pred.pred_GAT[i].load_state_dict(g["gat"][i])
            beh.behavior_encoder[i].load_state_dict(g["beh"][i])
            mac.agents[i].load_state_dict(g["actors"][i])
            mac.critics[i].load_state_dict(g["critics"][i])
        assert batch.packed is not None
        for t, st in enumerate(g["steps"]):
            pred.debug_gumbel = st["gumbel"].cuda().contiguous()
            att = pred.GAT_latent_update(st["history_single"], st["att_in"], st["beh_in"])
            d_att = maxdiff(att, st["att_out"])
            beh_now = st["beh_in"]
            d_beh = d_hid = 0.0
            if "beh_out" in st:
                beh_now, hid = beh.latent_update(st["window"], st["enc_rnn_in"], st["beh_in"])
                d_beh, d_hid = maxdiff(beh_now, st["beh_out"]), maxdiff(hid, st["enc_rnn_out"])
            batch.update({"avail_actions": g["avail"], "rnn_states_actors": st["rnn_a_in"],
                          "rnn_states_critics": st["rnn_c_in"], "history": st["history_single"],
                          "behavior_latent": st["beh_out"] if "beh_out" in st else st["beh_in"],
                          "attention_latent": st["att_out"]}, ts=t)
            # the packed rows must equal the reference's _build_inputs output
            F = mac.input_shape
            rows = batch.packed[:, :, t, :F].permute(1, 0, 2)
            d_in = maxdiff(rows, st["inputs"])
            mac.capture_logits = True
            values, actions, logps, rnn_a, rnn_c = mac.select_actions_ippo(batch, t_ep=t, test_mode=True)
            d_v = maxdiff(values, st["values"])
            d_lp = maxdiff(torch.cat(logps, dim=1), st["logp"].reshape(B, A))
            d_ra, d_rc = maxdiff(rnn_a, st["rnn_a_out"]), maxdiff(rnn_c, st["rnn_c_out"])
            print(f"[rollout {case} t={t}] att {d_att:.2e} beh {d_beh:.2e} hid {d_hid:.2e} in {d_in:.2e} "
                  f"val {d_v:.2e} logp {d_lp:.2e} rnn {d_ra:.2e}/{d_rc:.2e}")
            assert d_att < TOL and d_beh < TOL and d_hid < TOL and d_in < 1e-6
            assert d_v < TOL and d_lp < TOL and d_ra < TOL and d_rc < TOL
            assert (actions == st["actions"]).all()
            assert rnn_a.shape == st["rnn_a_out"].shape and values.shape == st["values"].shape
            batch.update({"actions": st["actions"]}, ts=t, mark_filled=False)


@pytest.mark.parametrize("B", [6, 3])
def test_gat_highway_shape_vs_oracle(B):
    """B envs (even / odd: the recurrence kernel packs two environments per CTA) x 5 agent-nets x 55 slots (Highway), seeded inputs, explicit noise:
    CUDA vs the CPU oracle.  Reports ill-conditioned edges (hard weight strictly inside
    (0.01, 0.99)) separately, as SURVEY §7 asks."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from oracle import iplan_oracle as O
    args = make_args("highway")
    A, N, o, L, D = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim
    torch.manual_seed(5)
    pred = Prediction_policy(args, None)
    params = [{k: v.detach().cpu().clone() for k, v in net.state_dict().items()} for net in pred.pred_GAT]
    rng = np.random.default_rng(3)
    hist = rng.uniform(-1, 1, size=(B, A, N, o)).astype(np.float32)
    hist[..., 0] = 1.0
    hist[:, :, 30:] = 0.0
    beh = rng.dirichlet(np.ones(L), size=(B, A, N)).astype(np.float32)
    att = rng.uniform(-1, 1, size=(B, A, N, D)).astype(np.float32)
    gum = torch.stack([O.draw_gumbel(B * N * (N - 1)).view(B, N, N - 1, 2) for _ in range(A)])
    ref = O.gat_latent_update(params, hist, att, beh, gum)
    pred.debug_gumbel = gum.cuda().contiguous()
    pred.capture_hard = True
    out = pred.GAT_latent_update(hist, att, beh)
    d = np.abs(out - ref.numpy())
    hard = pred.last_hard.cpu()
    frac_mid = float(((hard > 0.01) & (hard < 0.99)).float().mean())
    print(f"[gat highway] max {d.max():.3e} mean {d.mean():.3e} ill-conditioned edge fraction {frac_mid:.4f}")
    assert out.dtype == np.float32 and out.shape == (B, A, N, D)
    assert d.max() < TOL
    # production noise path: statistically the same gate-open rate as the parity path
    pred.debug_gumbel = None
    out2 = pred.GAT_latent_update(hist, att, beh)
    hard2 = pred.last_hard.cpu()
    assert np.isfinite(out2).all()
    assert abs(float(hard2.mean()) - float(hard.mean())) < 0.02


def test_behavior_and_controller_highway_shape_vs_oracle():
    _need_gpu()
    from iplan_b200.config import controller_input_dim, make_args
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from iplan_b200.nova.stable_behavior_policy import Behavior_policy
    from oracle import iplan_oracle as O
    args = make_args("highway")
    B, A, N, o, L, E, W = 19, args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, 32, args.max_history_len
    torch.manual_seed(11)
    beh = Behavior_policy(args, None)
    bp = [{k: v.detach().cpu().clone() for k, v in net.state_dict().items()} for net in beh.behavior_encoder]
    rng = np.random.default_rng(8)
    window = rng.uniform(-1, 1, size=(B, A, N, W, o))
    hid = rng.uniform(-1, 1, size=(B, 1, A, N, E)).astype(np.float32)
    prev = rng.dirichlet(np.ones(L), size=(B, A, N)).astype(np.float32)
    ref_lat, ref_hid = O.behavior_latent_update(bp, window, hid, prev)
    lat, new_hid = beh.latent_update(window, hid, prev)
    assert torch.is_tensor(new_hid) and tuple(new_hid.shape) == (B, 1, A, N, E)
    assert maxdiff(lat, ref_lat) < TOL and maxdiff(new_hid, ref_hid) < TOL

    scheme, groups, pre = make_scheme(args)
    from iplan_b200.components.episode_buffer import EpisodeBatch
    batch = EpisodeBatch(scheme, groups, B, 3, preprocess=pre, device="cuda")
    mac = DcntrlMAC(batch.scheme, groups, args)
    F = controller_input_dim(args)
    assert mac.input_shape == F == 2485
    with torch.no_grad():
        for net in mac.agents:
            net.act.action_out.linear.weight.mul_(50.0)
        mac.actor_stack.flat[:, :2 * F].uniform_(0.5, 1.5)        # feature_norm weight|bias away from (1, 0)
        mac.critic_stack.flat[:, :2 * F].uniform_(0.5, 1.5)
    ap = [{k: v.detach().cpu().clone() for k, v in n.state_dict().items()} for n in mac.agents]
    cp = [{k: v.detach().cpu().clone() for k, v in n.state_dict().items()} for n in mac.critics]
    x = torch.tensor(rng.uniform(-1, 1, size=(B, A, F)).astype(np.float32))
    x[..., 700:1500] = 0.0
    feat = x.permute(1, 0, 2).contiguous().cuda()
    ra = torch.tensor(rng.uniform(-1, 1, size=(B, A, 64)).astype(np.float32))
    rc_ = torch.tensor(rng.uniform(-1, 1, size=(B, A, 64)).astype(np.float32))
    avail = torch.ones(B, A, args.n_actions, dtype=torch.int64)
    avail[3, 1, 2] = 0
    uni = torch.tensor(rng.uniform(0, 1, size=(B, A)).astype(np.float32))
    ref = O.select_actions(ap, cp, x, avail, ra, rc_, test_mode=False, uniforms=uni)
    na, nc = torch.empty(A, B, 64, device="cuda"), torch.empty(A, B, 64, device="cuda")
    logits = torch.empty(A, B, args.n_actions, device="cuda")
    actions, logp, values = mac.controller_step(
        feat, ra.permute(1, 0, 2).contiguous().cuda(), rc_.permute(1, 0, 2).contiguous().cuda(), na, nc,
        (avail != 0).permute(1, 0, 2).contiguous().to(torch.uint8).cuda(), test_mode=False,
        uniforms=uni.t().contiguous().cuda(), logits=logits)
    torch.cuda.synchronize()
    keep = ref["logits"] > -1e9
    assert maxdiff(logits.permute(1, 0, 2).cpu()[keep], ref["logits"][keep]) < TOL
    assert maxdiff(values.t(), ref["values"]) < TOL
    assert maxdiff(na.permute(1, 0, 2), ref["rnn_a"]) < TOL and maxdiff(nc.permute(1, 0, 2), ref["rnn_c"]) < TOL
    same = (actions.t().cpu().long() == ref["actions"])
    assert same.float().mean() > 0.97          # a uniform within 1e-6 of a CDF edge may flip
    assert maxdiff(logp.t().cpu()[same], ref["logp"][same]) < TOL


def test_argument_checks_fail_loudly():
    _need_gpu()
    from iplan_b200 import _lib
    z = _lib.View(0, 0, 0, 0)
    rc = _lib.lib.iplan_gat_step(None, 0, z, z, z, z, None, 0, 0, 0.01, None, None, 0, 1, 1, 200, 5, 8, None)
    assert rc != 0 and b"n_slots" in _lib.lib.iplan_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc, "gat_step")


def test_device_resident_runner_equals_reference_api_path():
    """BASELINE configs[1] (Hetero-Highway mild, 5 agents, 64 envs, T = 90): the device-resident runner (kernels read
    and write the packed EpisodeBatch in place) and the reference's call pattern (numpy in / numpy out through
    GAT_latent_update / latent_update / EpisodeBatch.update / select_actions_ippo every timestep) are two hosts of the
    same kernels with the same Philox streams, so a whole greedy episode must agree: same actions, same stored
    latents / hidden states / one-hot columns."""
    _need_gpu()
    from iplan_b200.runners.synthetic_runner import build_system
    sa = build_system(n_envs=64, env="highway", hazard=0.002, seed=7)
    sb = build_system(n_envs=64, env="highway", hazard=0.002, seed=7)
    for x, y in ((sa.mac.actor_stack, sb.mac.actor_stack), (sa.prediction.stack, sb.prediction.stack),
                 (sa.behavior.stack, sb.behavior.stack)):
        assert torch.equal(x.flat, y.flat)
    ba, *_ = sa.runner.run(test_mode=True)
    bb, *_ = sb.runner.run_reference_api(test_mode=True)
    torch.cuda.synchronize()
    T = sa.args.episode_limit
    assert torch.equal(ba["actions"][:, :T], bb["actions"][:, :T])
    for key in ("attention_latent", "behavior_latent", "history", "rnn_states_actors", "rnn_states_critics"):
        d = maxdiff(ba[key], bb[key])
        print(f"[runner vs api] {key}: {d:.3e}")
        assert d <= 1e-6, (key, d)
    F = sa.mac.input_shape
    d = maxdiff(ba.packed[:, :, :T + 1, :F], bb.packed[:, :, :T + 1, :F])
    print(f"[runner vs api] packed controller rows: {d:.3e}")
    assert d <= 1e-6
    assert torch.equal(ba["terminated"][:, :T], bb["terminated"][:, :T]) and maxdiff(ba["reward"][:, :T], bb["reward"][:, :T]) == 0.0


def test_native_host_pipeline_equals_device_launches():
    """csrc/host_api.cu (iplan_gat_latent_update_host / iplan_behavior_latent_update_host: copy-in, kernel and copy-out
    pipelined over env pieces inside one native call) behind GAT_latent_update / latent_update at 130 envs (ragged pieces),
    with pageable and page-locked inputs and with arrays handed straight back (device shadows): bit-equal to launching the
    same kernels on device tensors piece by piece with the same noise counters."""
    _need_gpu()
    from iplan_b200 import _lib
    from iplan_b200.config import make_args
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from iplan_b200.nova.stable_behavior_policy import Behavior_policy
    args = make_args("highway", use_cuda=True, device="cuda")
    B, A, N, o, L, D, W = 130, args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim, args.max_history_len
    assert B >= _lib.PIPELINE_MIN_ROWS
    torch.manual_seed(11)
    pred, beh = Prediction_policy(args, None), Behavior_policy(args, None)
    rng = np.random.default_rng(5)
    perm = (1, 0, 2, 3)

    ends = _lib.wave_chunks(B, lambda e: (2 * e * A + 3) // 4)                   # the pieces the native call cuts the envs into

    def device_gat(hist, att, behl, calls0, n):
        assert n == len(ends)
        pred.calls = calls0
        h, a_, b_ = (torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).cuda() for x in (hist, att, behl))
        ref = torch.empty(B, A, N, D, device="cuda")
        for c in range(n):
            lo, hi = (ends[c - 1] if c else 0), ends[c]
            pred.gat_step(h[lo:hi].permute(perm), b_[lo:hi].permute(perm), a_[lo:hi].permute(perm), ref[lo:hi].permute(perm))
        return ref.cpu().numpy()

    hist = rng.uniform(-1, 1, size=(B, A, N, o))                          # float64, pageable: the reference's wrapper hands this over
    att = np.zeros((B, A, N, D), dtype=np.float32)
    behl = rng.dirichlet(np.ones(L), size=(B, A, N)).astype(np.float32)
    c0 = pred.calls
    out1 = pred.GAT_latent_update(hist, att, behl)
    n1 = pred.calls - c0
    assert n1 >= 2, "the native pipeline should cut 130 envs into pieces"
    ref1 = device_gat(hist, att, behl, c0, n1)
    assert np.array_equal(out1, ref1)
    # second call: the returned array handed straight back (device shadow, no upload), page-locked history
    hist2 = _lib.pinned_numpy(torch.as_tensor(rng.uniform(-1, 1, size=(B, A, N, o)), dtype=torch.float32))
    before = dict(_lib.io_bytes)
    c1 = pred.calls
    out2 = pred.GAT_latent_update(hist2, out1, behl)
    assert _lib.io_bytes["h2d_saved"] - before["h2d_saved"] == out1.nbytes
    assert np.array_equal(out2, device_gat(hist2, out1, behl, c1, pred.calls - c1))
    # behaviour encoder: deterministic, so one launch over all envs is the comparison
    win = rng.uniform(-1, 1, size=(B, A, N, W, o)).astype(np.float32)
    hid0 = rng.uniform(-1, 1, size=(B, 1, A, N, args.encoder_rnn_dim)).astype(np.float32)
    new1, hid1 = beh.latent_update(win, hid0, behl)
    w_d, p_d = torch.as_tensor(win).cuda(), torch.as_tensor(behl).cuda()
    h_d = torch.as_tensor(hid0).cuda().clone()
    n_d = torch.empty(B, A, N, L, device="cuda")
    beh.behavior_step(w_d.reshape(B, A, N, W * o).permute(perm), h_d[:, 0].permute(perm), p_d.permute(perm), n_d.permute(perm))
    assert np.array_equal(new1, n_d.cpu().numpy()) and torch.equal(hid1, h_d)
    new2, hid2 = beh.latent_update(win, hid1, new1)                       # shadowed latent + device hidden handed back
    n2 = torch.empty(B, A, N, L, device="cuda")
    beh.behavior_step(w_d.reshape(B, A, N, W * o).permute(perm), h_d[:, 0].permute(perm), n_d.permute(perm), n2.permute(perm))
    assert np.array_equal(new2, n2.cpu().numpy()) and torch.equal(hid2, h_d)


def test_obs_history_kernel_vs_reference_golden(golden_dir):
    """iplan_obs_history_step through the reference-named wrapper class: slot assignment in first-seen order, windows and
    newest rows bit-equal to the reference's wrapper over 14 recorded timesteps; the device window feeds K1b's layout."""
    _need_gpu()
    from iplan_b200.config import make_args
    from iplan_b200.observation_wrapper import observersation_state_history_wrapper as Wrapper
    g = load(golden_dir, "obs_wrapper.pt")
    d = g["dims"]
    args = make_args("highway", batch_size_run=d["B"], use_cuda=True, device="cuda")
    wr = Wrapper(args, d["A"], d["N"], args.episode_limit, d["W"])
    for t, st in enumerate(g["steps"]):
        obs = st["obs"].numpy()
        if t == 0:
            wr.agent_obs_profile_init(obs)
        wr.obs_history_create(obs)
        single, window = wr.obs_single_history_output(), wr.obs_history_output()
        assert single.dtype == np.float32 and window.shape == tuple(st["window"].shape)
        assert (single == st["single"].numpy()).all(), t
        assert (window == st["window"].numpy()).all(), t
    ids = wr.slot_ids.cpu()
    for k in range(d["B"]):
        for i in range(d["A"]):
            ref = g["ids"][k][i]
            assert ids[k, i, :len(ref)].tolist() == ref and int(wr.slot_count[k, i]) == len(ref)
    assert wr.window.view(d["B"], d["A"], d["N"], -1).permute(1, 0, 2, 3).stride(3) == 1      # K1b's [A,B,N,W*o] view
    # a second episode starts from a clean table
    wr.agent_obs_profile_init(g["steps"][0]["obs"].numpy())
    wr.obs_history_create(g["steps"][0]["obs"].numpy())
    assert (wr.obs_history_output() == g["steps"][0]["window"].numpy()).all()


def test_obs_wrapper_full_episode_vs_reference_wrapper(golden_dir):
    """A whole 91-observation episode (vehicles enter, leave and re-enter the agents' view; more observations than the
    deque's maxlen): every timestep's obs_single_history_output / obs_history_output and the final
    obs_history_episode_output(mask) bit-equal to the REFERENCE'S OWN wrapper (observation_wrapper.py) on the same inputs,
    recorded as digests of its float32 outputs in tests/golden/obs_wrapper_episode.json; the device `step()` hook returns
    the same tensors without a host copy."""
    _need_gpu()
    import json
    sys.path.insert(0, golden_dir)
    from obs_episode import f32_digest, obs_episode_inputs
    from iplan_b200.config import make_args
    from iplan_b200.observation_wrapper import observersation_state_history_wrapper as Wrapper
    with open(os.path.join(golden_dir, "obs_wrapper_episode.json")) as f:
        g = json.load(f)
    d = g["dims"]
    B, M = d["B"], d["M"]
    args = make_args("highway", batch_size_run=B, use_cuda=True, device="cuda")
    A, N, W, o, L = args.n_agents, args.max_vehicle_num, args.max_history_len, args.obs_shape_single, args.episode_limit
    assert (A, N, W, o, L) == (d["A"], d["N"], d["W"], d["o"], d["L"])
    own = Wrapper(args, A, N, L, W)
    own2 = Wrapper(args, A, N, L, W)                    # driven through the device hook
    steps, mask = obs_episode_inputs(np.random.default_rng(99), B, A, N, M, o, L)
    for t, obs32 in enumerate(steps):
        assert f32_digest(obs32) == g["obs"][t], t      # the recorded inputs
        if t == 0:
            own.agent_obs_profile_init(obs32)
        own.obs_history_create(obs32)
        s_dev, w_dev = own2.step(torch.as_tensor(obs32, dtype=torch.float32).cuda().contiguous())
        assert f32_digest(own.obs_single_history_output()) == g["single"][t], t
        assert f32_digest(own.obs_history_output()) == g["window"][t], t
        assert torch.equal(s_dev, own.single) and torch.equal(w_dev, own.window)
    for k in range(B):
        for i in range(A):
            assert own.slot_ids[k, i, :len(g["ids"][k][i])].tolist() == g["ids"][k][i]
    raw, ep = own.obs_history_episode_output(mask)
    assert f32_digest(raw) == g["raw"] and f32_digest(ep) == g["ep"]
