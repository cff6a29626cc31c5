"""Parity at the sizes BASELINE.json names (configs[1] = 64 envs, configs[2] = 512 envs; Hetero-Highway, 5 agents,
55 slots, T = 90): the kernels run at the full size — every grid-dependent path (two envs per CTA in K1, K1c's envs-per-CTA
wave, the row-chunk split of the fc1 backward) is exercised as in the benchmark — and a sub-sample (environments are
independent in the rollout; agents are independent in the update) is checked against the CPU oracle
(oracle/iplan_oracle.py, pinned to the reference by tests/test_oracle_golden.py) fed the same explicit noise.
Tolerance 1e-4 (north_star)."""
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


def _params(stack):
    return [{k: v.detach().cpu().clone() for k, v in n.state_dict().items()} for n in stack.nets]


@pytest.mark.parametrize("B,sample", [(64, (0, 33, 63)), (512, (1, 510))])
def test_whole_episode_device_runner_vs_oracle(B, sample):
    """The device-resident runner (`ParallelRunner.run`, the path bench.py times) over a WHOLE T = 90 episode at B envs,
    with the Gumbel noise of every K1 call and the sampling uniforms of every K1c call injected, against the oracle
    stepping the same episode for the sampled environments (reference call order,
    runners/ippo_parallel_runner.py:105-281): stored attention / behaviour latents, rnn states, actions, values, log-probs."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from iplan_b200.runners.synthetic_runner import build_system
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    sysm = build_system(n_envs=B, env="highway", hazard=0.01, seed=11 + B)
    a = sysm.args
    A, N, T = a.n_agents, a.max_vehicle_num, a.episode_limit
    with torch.no_grad():                                   # non-degenerate policy head (the 0.01-gain init is ~uniform)
        for ag in sysm.mac.agents:
            ag.act.action_out.linear.weight.mul_(30.0)
    S = list(sample)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(97 + B)
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
    worst, flips = oracle_episode(sysm, batch, S, rec)
    print(f"[episode B={B} envs {S}] worst |cuda - oracle| over {T} steps: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + f"; sampled actions differing: {flips} of {T * A * len(S)}")
    assert flips <= 1
    assert all(v < TOL for v in worst.values()), worst


def oracle_episode(sysm, batch, S, rec):
    """The oracle stepping the episode ``sysm.runner.run`` just ran, for the environments S, fed the noise of every K1
    call (rec["gumbel"][k]: [A, len(S), N, N-1, 2]) and K1c call (rec["uniforms"][t]: [A, len(S)]).  Returns the worst
    |CUDA - oracle| per quantity and the number of sampled actions that differ."""
    from oracle import iplan_oracle as O
    a = sysm.args
    A, N, T, W, nA = a.n_agents, a.max_vehicle_num, a.episode_limit, a.max_history_len, a.n_actions
    gat_p, beh_p = _params(sysm.prediction.stack), _params(sysm.behavior.stack)
    act_p, cri_p = _params(sysm.mac.actor_stack), _params(sysm.mac.critic_stack)
    hist = sysm.env.history[:, S].cpu()                     # [T+1, s, A, N, o]
    ns = len(S)
    att = torch.zeros(ns, A, N, a.attention_dim)
    beh = torch.zeros(ns, A, N, a.latent_dim)
    enc = torch.zeros(ns, 1, A, N, a.encoder_rnn_dim)
    rnn_a = torch.zeros(ns, A, a.rnn_hidden_dim)
    rnn_c = torch.zeros(ns, A, a.rnn_hidden_dim)
    last = torch.zeros(ns, A, nA)
    avail = torch.ones(ns, A, nA)

    def window(t):
        w = torch.zeros(ns, A, N, W, hist.shape[-1])
        lo = max(0, t - W + 1)
        w[:, :, :, W - (t - lo + 1):] = hist[lo:t + 1].permute(1, 2, 3, 0, 4)
        return w

    got = {k: batch[k][S].float().cpu() for k in ("attention_latent", "behavior_latent", "rnn_states_actors", "rnn_states_critics")}
    got_act = batch["actions"][S].cpu()[..., 0]
    got_val = sysm.runner.last_values[:, :, S].cpu()        # [T, A, s]
    got_lp = sysm.runner.last_logp[:, :, S].cpu()
    worst = dict(att=0.0, beh=0.0, rnn_a=0.0, rnn_c=0.0, value=0.0, logp=0.0)
    flips = 0
    with torch.no_grad():
        att = torch.as_tensor(O.gat_latent_update(gat_p, hist[0].numpy(), att.numpy(), beh.numpy(), rec["gumbel"][0]))
        worst["att"] = max(worst["att"], float((got["attention_latent"][:, 0] - att).abs().max()))
        for t in range(T):
            x = O.build_inputs_step(hist[t], att, beh, last, A)
            r = O.select_actions(act_p, cri_p, x, avail, rnn_a, rnn_c, uniforms=rec["uniforms"][t].t())
            worst["rnn_a"] = max(worst["rnn_a"], float((got["rnn_states_actors"][:, t] - rnn_a).abs().max()))
            worst["rnn_c"] = max(worst["rnn_c"], float((got["rnn_states_critics"][:, t] - rnn_c).abs().max()))
            worst["value"] = max(worst["value"], float((got_val[t].t() - r["values"]).abs().max()))
            same = got_act[:, t] == r["actions"]
            flips += int((~same).sum())
            # a uniform within fp32 noise of a CDF edge may pick the neighbouring action: follow the CUDA run's action so
            # that the rest of the episode stays comparable, and compare log-probs where the actions agree
            lp_o = torch.log_softmax(r["logits"], -1).gather(-1, got_act[:, t].unsqueeze(-1)).squeeze(-1)
            worst["logp"] = max(worst["logp"], float((got_lp[t].t() - lp_o).abs().max()))
            rnn_a, rnn_c = r["rnn_a"], r["rnn_c"]
            last = torch.nn.functional.one_hot(got_act[:, t], nA).float()
            att_new = torch.as_tensor(O.gat_latent_update(gat_p, hist[t + 1].numpy(), att.numpy(), beh.numpy(), rec["gumbel"][t + 1]))
            beh_new, enc_new = O.behavior_latent_update(beh_p, window(t + 1).numpy(), enc.numpy(), beh.numpy(), a.soft_update_coef)
            att, beh, enc = att_new, torch.as_tensor(beh_new), torch.as_tensor(enc_new)
            worst["att"] = max(worst["att"], float((got["attention_latent"][:, t + 1] - att).abs().max()))
            worst["beh"] = max(worst["beh"], float((got["behavior_latent"][:, t + 1] - beh).abs().max()))
    return worst, flips


def test_learner_vs_oracle_baseline_shape():
    """IPPOLearner.train at Bf = 64 full-length episodes (T = 90), 15 epochs, 5 agents — the update of configs[1] — on the
    CUDA path; agent 3 is re-trained by the oracle (autograd + Adam on the CPU) from the same data and weights: pre-update
    returns / advantages / values / old log-probs, first-epoch gradients and the post-update weights."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib.util
    spec = importlib.util.spec_from_file_location("test_gpu_learner", os.path.join(ROOT, "tests", "test_gpu_learner.py"))
    tgl = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tgl)
    build = tgl.build
    from iplan_b200.config import make_args
    from iplan_b200.modules.flat import ParamStack
    from oracle import iplan_oracle as O
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    B = 64
    args = make_args("highway", batch_size_run=B, buffer_size=B, batch_size=B - 1, use_cuda=True, device="cuda")
    A, N, o, L, D, R, T = args.n_agents, args.max_vehicle_num, args.obs_shape_single, args.latent_dim, args.attention_dim, args.rnn_hidden_dim, args.episode_limit
    rng = np.random.default_rng(17)
    hist = rng.uniform(-1, 1, size=(B, T + 1, A, N, o)).astype(np.float32)
    hist[..., 0] = 1.0
    for t in range(T + 1):
        hist[:, t, :, min(N, 15 + t // 3):] = 0.0
    term = (np.cumsum(rng.uniform(size=(B, T + 1, A, 1)) < 0.01, axis=1) > 0).astype(np.uint8)
    data = dict(history=hist, attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
                behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
                rnn_states_actors=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                rnn_states_critics=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                actions=rng.integers(0, 5, size=(B, T + 1, A, 1)), avail_actions=np.ones((B, T + 1, A, 5), dtype=np.int64),
                reward=(rng.normal(size=(B, T + 1, A, 1)) * 2).astype(np.float32), terminated=term)
    torch.manual_seed(5)
    F = N * (o + D + L) + 5 + A
    a0, c0 = ParamStack("actor", A, (F, 5)), ParamStack("critic", A, (F,))
    with torch.no_grad():
        for n in a0.nets:
            n.act.action_out.linear.weight.mul_(30.0)
    actors = [{k: v.clone() for k, v in n.state_dict().items()} for n in a0.nets]
    critics = [{k: v.clone() for k, v in n.state_dict().items()} for n in c0.nets]
    batch, mac, learner, log = build(args, data, actors, critics)
    learner.keep_pre = True
    learner.insert_episode_batch(batch)
    learner.train(0)
    torch.cuda.synchronize()
    ag = 3
    dt = {k: torch.as_tensor(v) for k, v in data.items()}
    onehot = torch.nn.functional.one_hot(dt["actions"].squeeze(-1), 5).float()
    ob = dict(history=dt["history"][:, :, ag], attention_latent=dt["attention_latent"][:, :, ag],
              behavior_latent=dt["behavior_latent"][:, :, ag], actions=dt["actions"][:, :, ag],
              actions_onehot=onehot[:, :, ag], available_actions=dt["avail_actions"][:, :, ag],
              reward=dt["reward"][:, :, ag], terminated_masks=(1 - dt["terminated"][:, :, ag].float()),
              rnn_states_actor=dt["rnn_states_actors"][:, :, ag], rnn_states_critic=dt["rnn_states_critics"][:, :, ag])
    ap = {k: v.clone() for k, v in actors[ag].items()}
    cp = {k: v.clone() for k, v in critics[ag].items()}
    T_, nb_ = args.episode_limit, args.batch_size
    perms = [torch.randperm(nb_ * T_, generator=torch.Generator().manual_seed(100 + e)) for e in range(args.ppo_epoch)]
    stats, pre, _, _ = O.train_agent(ap, cp, ob, ag, SimpleNamespace(**vars(args)), perms=perms)
    # the same update in fp64 (same row order): how far fp32 arithmetic itself moves the post-update weights.  Fifteen Adam
    # steps divide every gradient by sqrt(v) + 1e-5, so a weight whose gradient sits at the rounding floor can move by a
    # fraction of lr = 5e-4 between two correct fp32 evaluations; that conditioning, not 1e-4, is the yardstick below.
    dbl = lambda d: {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}
    ap64, cp64 = dbl({k: v.clone() for k, v in actors[ag].items()}), dbl({k: v.clone() for k, v in critics[ag].items()})
    O.train_agent(ap64, cp64, dbl(ob), ag, SimpleNamespace(**vars(args)), perms=perms)
    mine = learner.last_pre
    dpre = {k: float((mine[k][ag].cpu().double() - pre[k].double()).abs().max()) for k in ("values_all", "returns", "advantages", "old_logp")}
    offs = {"actor": mac.actor_stack.named_offsets(), "critic": mac.critic_stack.named_offsets()}
    worst_grad = 0.0
    for kind, key in (("actor", "grads_actor"), ("critic", "grads_critic")):
        for name, gref in stats[0][key].items():
            off, shape = offs[kind][name]
            gm = learner.first_grads[kind][ag, off:off + gref.numel()].view(gref.shape).cpu()
            worst_grad = max(worst_grad, float((gm - gref).abs().max() / (gref.abs().max() + 1e-12)))
    worst_w, n_off, n_all, ref_w, ref_off = 0.0, 0, 0, 0.0, 0
    sq_dev, sq_ref, sq_moved = 0.0, 0.0, 0.0
    for kind, nets, ref, ref64, init in (("actor", mac.agents, ap, ap64, actors[ag]), ("critic", mac.critics, cp, cp64, critics[ag])):
        sd = nets[ag].state_dict()
        for k, v in ref.items():
            d = (sd[k].detach().cpu().double() - ref64[k].detach().double()).abs()           # CUDA vs the fp64 oracle
            r = (v.detach().double() - ref64[k].detach().double()).abs()                     # fp32 oracle vs the fp64 oracle
            mv = (ref64[k].detach().double() - init[k].detach().double())                    # how far the update moved the weight
            worst_w = max(worst_w, float(d.max()) if d.numel() else 0.0)
            ref_w = max(ref_w, float(r.max()) if r.numel() else 0.0)
            n_off += int((d > 5e-5).sum())
            ref_off += int((r > 5e-5).sum())
            n_all += d.numel()
            sq_dev += float((d * d).sum()); sq_ref += float((r * r).sum()); sq_moved += float((mv * mv).sum())
    rms_dev, rms_ref, rms_moved = (sq_dev / n_all) ** 0.5, (sq_ref / n_all) ** 0.5, (sq_moved / n_all) ** 0.5
    print(f"[learner Bf=64 T=90 15 epochs, agent {ag}] pre {dpre}; worst first-epoch grad rel {worst_grad:.2e}; post-train weights vs the fp64 "
          f"oracle: CUDA worst {worst_w:.2e}, rms {rms_dev:.2e}, {n_off} of {n_all} off by > 5e-5; fp32 oracle worst {ref_w:.2e}, rms {rms_ref:.2e}, "
          f"{ref_off} off by > 5e-5; rms movement of the weights over the update {rms_moved:.2e}")
    assert all(v < 2e-4 for v in dpre.values()), dpre
    # same weights, same data: the first epoch's gradients are the parity statement proper
    assert worst_grad < 1e-5
    # After fifteen Adam steps the comparison is one of conditioning, not of arithmetic: PPO's ratio clip, the value clip and the
    # Huber switch are discontinuous per sample, and Adam divides by sqrt(v) + 1e-5, so two correct fp32 evaluations of the
    # same update already differ from the fp64 one by a few 1e-5 on isolated weights (the fp32 oracle's own numbers are
    # printed above; they change with the host's thread count).  What is asserted: the CUDA weights stay within one learning
    # rate of the fp64 result everywhere, within 2 % of the update's own size in the rms sense, and all but 0.5 % of them
    # within 5e-5.
    assert worst_w < args.lr
    assert rms_dev < 0.02 * rms_moved
    assert n_off <= 0.005 * n_all


def test_fc1_at_bench_shape():
    """tools/check_fc1.py at the benchmark's shape (5 agents x 46 592 rows = 512 envs x 91 x 2 496 features): the fc1
    forward / backward against an fp64 reference."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib.util
    spec = importlib.util.spec_from_file_location("check_fc1", os.path.join(ROOT, "tools", "check_fc1.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.run(5, 46592, 2485, reps=1) < 1e-5
