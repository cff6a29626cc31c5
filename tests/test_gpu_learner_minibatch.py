"""IPPOLearner.train with num_mini_batch > 1 on the device.

 (1) against the reference's own learner run with num_mini_batch = 3 (tests/golden/learner_minibatch.pt), its
     permutations injected through ``learner.debug_perm``: post-update weights and the six statistics;
 (2) against the float64 oracle at the benchmark's learner shape (Highway, 512 episodes, T = 90, F = 2485) for
     num_mini_batch 2, 4 and 7, every mini-batch of the first and the last epoch in lockstep, with the machinery of
     test_gpu_learner_epochs.py (the Adam tap, the branch-edge and ReLU-kink allowances, its tolerances): gradients,
     the loss / entropy / ratio sums, the gradient norms, clip + Adam on the CUDA (p, g, m, v).  No mini-batch is a
     whole number of 128-row tiles, and 4 does not divide 45 990: its two trailing rows are dropped;
 (3) two train() calls from equal weights, inputs and permutations give bit-equal parameters (1 and 4 mini-batches);
     with num_mini_batch = 1 no permutation is drawn and no gathered copy is allocated;
 (4) the saved Adam step advances ppo_epoch * num_mini_batch per train(); generate_data yields the sets' rows;
 (5) two GPUs (skipped with fewer): two ranks with 4 mini-batches equal one rank on the concatenated batch."""
import importlib.util
import os
import socket
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _mod(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _golden(golden_dir):
    from tests.golden.minibatch_fixture import load
    return load(os.path.join(golden_dir, "learner_minibatch.pt"))


def _golden_learner(g, **over):
    from tests.test_gpu_rollout import args_from
    tgl = _mod("test_gpu_learner")
    args = args_from(dict(g["args"], **over))
    batch, mac, learner, log = tgl.build(args, g["data"], g["actors_before"], g["critics_before"])
    learner.insert_episode_batch(batch)
    return args, batch, mac, learner


def test_train_matches_reference_golden(golden_dir):
    g = _golden(golden_dir)
    args, batch, mac, learner = _golden_learner(g)
    assert learner.num_mini_batch == 3
    learner.debug_perm = g["perms"]
    learner.train(t_env=0)
    torch.cuda.synchronize()
    assert learner.debug_perm is None
    worst = 0.0
    for a in range(args.n_agents):
        for nets, after in ((mac.agents, g["actors_after"]), (mac.critics, g["critics_after"])):
            sd = nets[a].state_dict()
            worst = max([worst] + [float((sd[k].cpu() - v).abs().max()) for k, v in after[a].items()])
    moved = max(float((mac.agents[0].state_dict()[k].cpu() - v).abs().max()) for k, v in g["actors_before"][0].items())
    print(f"[minibatch golden] largest weight diff {worst:.2e} (weights moved by up to {moved:.2e})")
    assert worst < 1e-4 and moved > 1e-3
    for key in ("value_loss", "policy_loss", "dist_entropy", "actor_grad_norm", "critic_grad_norm", "ratio"):
        ref = [v for k, v in g["stats"].items() if k.endswith(key)][0]
        assert abs(learner.train_info[key] - ref) < 1e-4 * max(1.0, abs(ref)), (key, learner.train_info[key], ref)
    # the optimiser checkpoint carries the reference's step count
    assert int(learner.actor_optimizers[0].state_dict()["state"][0]["step"]) == g["opt_step"] == args.ppo_epoch * 3


@pytest.mark.parametrize("k", [2, 4, 7])
def test_mini_batches_at_bench_shape_against_float64(k, monkeypatch):
    from iplan_b200 import _lib
    from oracle import iplan_oracle as O
    E = _mod("test_gpu_learner_epochs")
    tgl = _mod("test_gpu_learner")
    dev = torch.device("cuda")
    args, data, actors, critics = E._highway_case(512, seed=23, num_mini_batch=k)
    batch, mac, learner, log = tgl.build(args, data, actors, critics)
    learner.keep_pre = True
    learner.insert_episode_batch(batch)
    A, T, nb = args.n_agents, args.episode_limit, args.batch_size
    n = nb * T
    mbs = n // k
    assert n == 45990 and mbs % 128 != 0 and (k != 4 or n % k == 2)
    gen = torch.Generator().manual_seed(100 + k)
    perms = torch.stack([torch.randperm(n, generator=gen) for _ in range(A * args.ppo_epoch)]).view(A, args.ppo_epoch, n)
    learner.debug_perm = perms
    perms = perms.to(dev)
    offs = {"actor": mac.actor_stack.named_offsets(), "critic": mac.critic_stack.named_offsets()}
    keys = {"actor": O.ACTOR_TRAINABLE, "critic": O.CRITIC_TRAINABLE}
    rows_base = [E._agent_rows(O, data, a, args, dev) for a in range(A)]
    oargs = SimpleNamespace(**vars(args))
    checked = (0, args.ppo_epoch - 1)
    state = dict(step=0, prev=None, fails=[], worst={})

    def unflat(vec, kind):
        return {key: vec[off:off + (int(np.prod(shape)) if len(shape) else 1)].view(shape).double().clone()
                for key, (off, shape) in offs[kind].items() if key in keys[kind]}

    def note(name, val, bound, where):
        state["worst"][name] = max(state["worst"].get(name, 0.0), val / bound)
        if not val <= bound:
            state["fails"].append(f"{where} {name}: {val:.3e} > {bound:.3e}")

    def on_set(ra, rc):
        ep, m = divmod(state["step"], k)
        state["step"] += 1
        prev = state["prev"] if state["prev"] is not None else torch.zeros_like(ra["stats"])
        state["prev"] = rc["stats_after"]
        if ep not in checked:
            return
        pre, gs = learner.last_pre, learner.grad_scale
        assert gs == 2.0 ** int(np.ceil(np.log2(mbs)))          # the pre-scale follows the mini-batch size
        for a in range(A):
            where = f"[k={k} epoch {ep} set {m} agent {a}]"
            idx = perms[a, ep, m * mbs:(m + 1) * mbs]
            full = dict(rows_base[a], ret=pre["returns"][a, :nb].reshape(-1).double(), old_lp=pre["old_logp"][a, :nb].reshape(-1).double(),
                        adv=pre["advantages"][a, :nb].reshape(-1).double(), old_v=pre["values_all"][a, :nb, :T].reshape(-1).double())
            flat = {key: v[idx] for key, v in full.items()}
            ap, cp = unflat(ra["p"][a], "actor"), unflat(rc["p"][a], "critic")
            e = O.ppo_epoch(ap, cp, flat, oargs, rows_out=True)
            f32 = lambda d: {key: (v.float() if v.is_floating_point() else v) for key, v in d.items()}
            e32 = O.ppo_epoch(f32(ap), f32(cp), f32(flat), oargs)
            ratio_edge, value_edge = E._edges(e, flat, args)
            flagged = {"actor": ratio_edge.nonzero().view(-1), "critic": value_edge.nonzero().view(-1)}
            for kind, rec in (("actor", ra), ("critic", rc)):
                assert flagged[kind].numel() <= max(8, E.MAX_FLAGGED * mbs), (where, kind, flagged[kind].numel())
                jump = E._jump_bound(O, ap, cp, flat, flagged[kind], kind, args)
                n_relu = E._relu_jump(O, ap if kind == "actor" else cp, flat, kind, e, jump)
                assert n_relu <= max(8, E.MAX_FLAGGED * mbs), (where, kind, "ReLU inputs near 0", n_relu)
                for key in keys[kind]:
                    off, shape = offs[kind][key]
                    ref = e["grads_" + kind][key]
                    got = rec["g"][a, off:off + ref.numel()].view(ref.shape).double() / gs
                    scale = max(float(ref.abs().max()), 3 * float((e32["grads_" + kind][key].double() - ref).abs().max()) / E.GRAD_TOL) + 1e-30
                    # The critic's two head-bias gradients are the open finding test_gpu_learner_epochs.py records for late
                    # epochs (above 1e-5 of their scale with no row near a branch edge; held to 5e-5 there): seen here at
                    # 1.16e-5 in one of the 70 checked mini-batches of num_mini_batch = 7 (epoch 14).  Same bound, these two only.
                    tol = 5e-5 if kind == "critic" and key in ("v_out.bias", "rnn.norm.bias") else E.GRAD_TOL
                    note("grad", float(((got - ref).abs() - jump[key]).max()) / scale, tol, f"{where} {kind}:{key}")
            dstat = (ra["stats"][a] - prev[a]).double()
            for col, key in ((0, "policy_loss"), (1, "value_loss"), (2, "dist_entropy"), (3, "ratio")):
                ref = float(e[key])
                note("stat", abs(float(dstat[col]) - ref) / max(1e-2, abs(ref)), E.STAT_TOL, f"{where} {key}")
            for kind, rec, col in (("actor", ra, 4), ("critic", rc, 5)):
                mask = learner.masks[kind] > 0
                g = rec["g"][a].double() / gs
                p, mm, v = rec["p"][a].double()[mask], rec["m"][a].double()[mask], rec["v"][a].double()[mask]
                gm, p0, m0 = g[mask], p.clone(), mm.clone()
                n64 = float(O.clip_adam_step([p], [gm], [mm], [v], rec["step"], rec["lr"], learner.optim_eps, learner.max_grad_norm,
                                             b1=float(np.float32(0.9)), b2=float(np.float32(0.999))))
                assert rec["step"] == ep * k + m + 1
                note("adam", abs(float(rec["sq"][a].double().sqrt()) - n64) / n64, 1e-6, f"{where} {kind} norm")
                note("stat", abs(float((rec["stats_after"][a, col] - rec["stats"][a, col]).double()) - n64) / max(1e-2, n64),
                     E.STAT_TOL, f"{where} {kind}_grad_norm")
                coef = min(1.0, learner.max_grad_norm / (n64 + 1e-6))
                mc, vc, pc = (rec[x][a].double()[mask] for x in ("m_after", "v_after", "p_after"))
                note("adam", float(((mc - mm).abs() / (0.9 * m0.abs() + 0.1 * coef * gm.abs() + 1e-30)).max()), 1e-6, f"{where} {kind} m")
                note("adam", float(((vc - v).abs() / (v + 1e-30)).max()), 1e-6, f"{where} {kind} v")
                ulp = torch.finfo(torch.float32).eps * p0.abs()
                note("adam", float(((pc - p).abs() / (4 * ulp + 1e-5 * rec["lr"])).max()), 1.0, f"{where} {kind} p")

    monkeypatch.setattr(_lib, "lib", E.AdamTap(_lib.lib, learner, on_set))
    learner.train(0)
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert state["step"] == args.ppo_epoch * k
    print(f"[minibatch k={k}] worst / bound: " + " ".join(f"{key} {v:.2f}" for key, v in state["worst"].items()))
    assert not state["fails"], "\n".join(state["fails"][:20])


@pytest.mark.parametrize("k", [1, 4])
def test_same_permutations_give_bit_equal_parameters(golden_dir, k):
    g = _golden(golden_dir)
    n = g["args"]["batch_size"] * g["args"]["episode_limit"]
    gen = torch.Generator().manual_seed(5)
    A, epochs = g["args"]["n_agents"], g["args"]["ppo_epoch"]
    perms = torch.stack([torch.randperm(n, generator=gen) for _ in range(A * epochs)]).view(A, epochs, n)
    out = []
    for _ in range(2):
        args, batch, mac, learner = _golden_learner(g, num_mini_batch=k)
        if k > 1:
            learner.debug_perm = perms.clone()
        state = learner.perm_gen.get_state()
        learner.train(0)
        torch.cuda.synchronize()
        if k == 1:      # the untouched path: nothing drawn, no gathered copy, the work buffers it always had
            assert torch.equal(learner.perm_gen.get_state(), state) and learner.mb is None
            assert sorted(learner.work) == sorted(
                ["key", "stat", "Wh", "Wl", "ws", "cc", "Z1", "Xh", "Xl", "Dh", "Dl", "gscale", "A1", "Z2", "A2", "GI", "GH", "SM", "G",
                 "logp", "ent", "value", "returns", "adv", "moments", "norm", "stats", "sq", "grads", "old_logp", "old_value"])
        else:
            assert learner.mb is not None and learner.mb["Xh"].numel() == A * (n // k) * learner.store["X"].shape[-1]
        out.append((mac.actor_stack.flat.clone(), mac.critic_stack.flat.clone(), dict(learner.train_info)))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]


def test_checkpoint_step_and_drawn_permutations(golden_dir, tmp_path):
    g = _golden(golden_dir)
    args, batch, mac, learner = _golden_learner(g, num_mini_batch=4, seed=11)
    learner.train(0)                                   # permutations drawn from the learner's own generator
    torch.cuda.synchronize()
    learner.save_models(str(tmp_path))
    for name in ("actor_0_opt.th", f"critic_{args.n_agents - 1}_opt.th"):
        sd = torch.load(os.path.join(str(tmp_path), name), weights_only=False)
        assert {int(s["step"]) for s in sd["state"].values()} == {args.ppo_epoch * 4}
    n = args.batch_size * args.episode_limit
    ref = torch.Generator().manual_seed(11)
    [torch.randperm(n, generator=ref) for _ in range(args.n_agents * args.ppo_epoch)]
    assert torch.equal(learner.perm_gen.get_state(), ref.get_state())
    with pytest.raises(ValueError):
        _golden_learner(g, num_mini_batch=n + 1)


def test_generate_data_yields_the_sets_rows(golden_dir):
    g = _golden(golden_dir)
    args, batch, mac, learner = _golden_learner(g)
    B, T, nA = args.buffer_size, args.episode_limit, args.n_actions
    row = torch.arange(B * T, dtype=torch.float32).view(B, T, 1)
    av = torch.arange(B * T).view(B, T, 1).expand(B, T, nA)
    perm = g["perms"][0, 1]
    out = list(learner.generate_data(row * 2, row, row, row.long(), row, row, row, row, av, row, num_mini_batch=3, perm=perm))
    mbs = perm.shape[0] // 3
    assert len(out) == 3
    for m, sample in enumerate(out):
        want = perm[m * mbs:(m + 1) * mbs].to("cuda")
        assert len(sample) == 10 and all(t.is_cuda and t.shape[0] == mbs for t in sample)
        assert torch.equal(sample[0][:, 0].long(), 2 * want) and torch.equal(sample[3][:, 0], want)
        assert all(torch.equal(t[:, 0].long(), want) for t in sample[1:])
    state = learner.perm_gen.get_state()
    drawn = next(learner.generate_data(row, row, row, row.long(), row, row, row, row, None, row, num_mini_batch=3))
    assert drawn[9] is None and not torch.equal(learner.perm_gen.get_state(), state)


# ---- two GPUs ----------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from iplan_b200.config import make_args
    from iplan_b200.modules.flat import ParamStack
    from tests.test_gpu_learner import build
    from tests.test_gpu_multi import _data
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        Bg, T, A, N = 16, 7, 5, 55
        data = _data(Bg, T, A, N)
        torch.manual_seed(4)
        F = N * 45 + 10
        a0, c0 = ParamStack("actor", A, (F, 5)), ParamStack("critic", A, (F,))
        actors = [{k: v.clone() for k, v in n.state_dict().items()} for n in a0.nets]
        critics = [{k: v.clone() for k, v in n.state_dict().items()} for n in c0.nets]
        Bl = Bg // world
        common = dict(episode_limit=T, ppo_epoch=3, use_cuda=True, device="cuda", batch_size=Bg - 1, num_mini_batch=4, seed=3)
        shard = {k: v[rank * Bl:(rank + 1) * Bl] for k, v in data.items()}
        batch, mac, learner, _ = build(make_args("highway", buffer_size=Bl, batch_size_run=Bl, **common), shard, actors, critics)
        learner.insert_episode_batch(batch)
        learner.train(0)
        torch.cuda.synchronize()
        res = {}
        if rank == 0:
            batch2, mac2, learner2, _ = build(make_args("highway", buffer_size=Bg, batch_size_run=Bg, **common), data, actors, critics)
            learner2.use_dist = False
            learner2.insert_episode_batch(batch2)
            learner2.train(0)
            torch.cuda.synchronize()
            rel = lambda x, y: float((x - y).abs().max() / y.abs().max())
            res = dict(da=rel(mac.actor_stack.flat, mac2.actor_stack.flat), dc=rel(mac.critic_stack.flat, mac2.critic_stack.flat),
                       info=learner.train_info, info2=learner2.train_info)
        w = mac.actor_stack.flat.clone()
        dist.broadcast(w, 0)
        res["rank_spread"] = float((w - mac.actor_stack.flat).abs().max())
        out.put(res)
    finally:
        dist.destroy_process_group()


def test_two_gpu_mini_batches_equal_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    r0 = [r for r in res if "da" in r][0]
    assert all(r["rank_spread"] == 0.0 for r in res)
    assert r0["da"] < 1e-5 and r0["dc"] < 1e-5, r0
    for key, v in r0["info2"].items():
        assert abs(r0["info"][key] - v) < 1e-4 * max(1.0, abs(v)), key
