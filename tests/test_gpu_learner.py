"""Parity of the CUDA learner (K2a GAE/advantage moments, fused forward, K2b PPO losses +
backward, fc1 products, clip + Adam) through IPPOLearner.insert_episode_batch / train against
 (1) the golden post-update weights and logged statistics produced by the reference's own
     IPPOLearner.train (tests/golden/learner.pt), and
 (2) the CPU oracle at a larger, Highway-shaped case."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.test_gpu_rollout import args_from, load, make_scheme, maxdiff

pytestmark = pytest.mark.gpu


class Log:
    def __init__(self):
        self.stats = {}

    def log_stat(self, k, v, t):
        self.stats[k] = float(v)


def build(args, data, actors, critics):
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from iplan_b200.learners.ippo_learner import IPPOLearner
    scheme, groups, pre = make_scheme(args)
    B = data["history"].shape[0]
    batch = EpisodeBatch(scheme, groups, B, args.episode_limit + 1, preprocess=pre, device="cuda")
    mac = DcntrlMAC(batch.scheme, groups, args)
    for i in range(args.n_agents):
        mac.agents[i].load_state_dict(actors[i])
        mac.critics[i].load_state_dict(critics[i])
    log = Log()
    learner = IPPOLearner(mac, batch.scheme, log, args)
    batch.update(data, bs=slice(None), ts=slice(None))
    return batch, mac, learner, log


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_train_matches_reference_golden(golden_dir, case):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    g = load(golden_dir, "learner.pt")[case]
    args = args_from(g["args"])
    A, T = args.n_agents, args.episode_limit
    batch, mac, learner, log = build(args, g["data"], g["actors_before"], g["critics_before"])
    # packed rows == the reference's _build_inputs_ippo output
    F = mac.input_shape
    for a in range(A):
        assert maxdiff(batch.packed[a, :, :, :F], g["pre"][a]["obs_all"]) < 1e-6
    learner.keep_pre = True
    learner.insert_episode_batch(batch)
    assert learner.can_sample()
    learner.train(t_env=0)
    torch.cuda.synchronize()
    pre = learner.last_pre
    worst = {}
    for a in range(A):
        ref = g["pre"][a]
        for k in ("values_all", "returns", "advantages", "old_logp"):
            worst[k] = max(worst.get(k, 0.0), maxdiff(pre[k][a], ref[k]))
    print(f"[learner {case}] pre-update diffs {worst}")
    assert worst["values_all"] < 1e-4 and worst["old_logp"] < 1e-4
    assert worst["returns"] < 2e-4 and worst["advantages"] < 2e-4
    dmax = {}
    for a in range(A):
        for kind, nets, after in (("actor", mac.agents, g["actors_after"]), ("critic", mac.critics, g["critics_after"])):
            sd = nets[a].state_dict()
            for k, v in after[a].items():
                d = maxdiff(sd[k], v)
                dmax[kind + ":" + k] = max(dmax.get(kind + ":" + k, 0.0), d)
    top = sorted(dmax.items(), key=lambda kv: -kv[1])[:5]
    print(f"[learner {case}] largest post-train weight diffs: {top}")
    # 15 (4) Adam steps of lr 5e-4 move a weight by <= 7.5e-3 (2e-3); agreement to 5e-5 abs
    assert top[0][1] < 5e-5, top
    for key in ("value_loss", "policy_loss", "dist_entropy", "actor_grad_norm", "critic_grad_norm", "ratio"):
        ref = [v for k, v in g["stats"].items() if k.endswith(key)][0]
        mine = learner.train_info[key]
        print(f"[learner {case}] {key}: cuda {mine:.6f} reference {ref:.6f}")
        assert abs(mine - ref) < 2e-4 * max(1.0, abs(ref)), (key, mine, ref)
    assert learner.count == 0 and not learner.can_sample()
    # optimiser checkpoint has the reference's structure: 18 tensors with Adam state
    sd = learner.actor_optimizers[0].state_dict()
    assert len(sd["state"]) == g["actor_opt_steps"][0] and len(sd["param_groups"][0]["params"]) == 22


def test_train_vs_oracle_highway_shape():
    """Full Highway dims (A=5, N=55, F=2485), Bf=12 episodes x T=9, 3 epochs: CUDA vs oracle."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from iplan_b200.config import make_args
    from oracle import iplan_oracle as O
    args = make_args("highway", episode_limit=9, buffer_size=12, batch_size=11, batch_size_run=12, ppo_epoch=3,
                     use_cuda=True, device="cuda")
    A, N, o, L, D, R, T, B = args.n_agents, args.max_vehicle_num, 5, 8, 32, 64, 9, 12
    rng = np.random.default_rng(5)
    hist = rng.uniform(-1, 1, size=(B, T + 1, A, N, o)).astype(np.float32)
    hist[..., 0] = 1.0
    hist[:, :, :, 25:] = 0.0
    term = np.zeros((B, T + 1, A, 1), dtype=np.uint8)
    term[2, 5:, 1] = 1
    term[7, 3:, 4] = 1
    data = dict(history=hist, attention_latent=rng.uniform(-1, 1, size=(B, T + 1, A, N, D)).astype(np.float32),
                behavior_latent=rng.dirichlet(np.ones(L), size=(B, T + 1, A, N)).astype(np.float32),
                rnn_states_actors=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                rnn_states_critics=rng.uniform(-1, 1, size=(B, T + 1, A, R)).astype(np.float32),
                actions=rng.integers(0, 5, size=(B, T + 1, A, 1)), avail_actions=np.ones((B, T + 1, A, 5), dtype=np.int64),
                reward=(rng.normal(size=(B, T + 1, A, 1)) * 2).astype(np.float32), terminated=term)
    torch.manual_seed(3)
    from iplan_b200.modules.flat import ParamStack
    F = N * 45 + 10
    a0 = ParamStack("actor", A, (F, 5))
    c0 = ParamStack("critic", A, (F,))
    with torch.no_grad():
        for n in a0.nets:
            n.act.action_out.linear.weight.mul_(30.0)
        a0.flat[:, :2 * F].uniform_(0.5, 1.5)
        c0.flat[:, :2 * F].uniform_(0.5, 1.5)
    actors = [{k: v.clone() for k, v in n.state_dict().items()} for n in a0.nets]
    critics = [{k: v.clone() for k, v in n.state_dict().items()} for n in c0.nets]
    batch, mac, learner, log = build(args, data, actors, critics)
    learner.keep_pre = True
    learner.insert_episode_batch(batch)
    learner.train(0)
    torch.cuda.synchronize()
    dt = {k: torch.as_tensor(v) for k, v in data.items()}
    onehot = torch.nn.functional.one_hot(dt["actions"].squeeze(-1), 5).float()
    oargs = SimpleNamespace(**vars(args))
    worst, worst_grad, n_off, n_all = 0.0, 0.0, 0, 0
    offs = {"actor": mac.actor_stack.named_offsets(), "critic": mac.critic_stack.named_offsets()}
    for a in range(A):
        ob = dict(history=dt["history"][:, :, a], attention_latent=dt["attention_latent"][:, :, a],
                  behavior_latent=dt["behavior_latent"][:, :, a], actions=dt["actions"][:, :, a],
                  actions_onehot=onehot[:, :, a], available_actions=dt["avail_actions"][:, :, a],
                  reward=dt["reward"][:, :, a], terminated_masks=(1 - dt["terminated"][:, :, a].float()),
                  rnn_states_actor=dt["rnn_states_actors"][:, :, a], rnn_states_critic=dt["rnn_states_critics"][:, :, a])
        ap = {k: v.clone() for k, v in actors[a].items()}
        cp = {k: v.clone() for k, v in critics[a].items()}
        stats, pre, _, _ = O.train_agent(ap, cp, ob, a, oargs)
        mine = learner.last_pre
        dpre = {k: maxdiff(mine[k][a], pre[k]) for k in ("values_all", "returns", "advantages", "old_logp")}
        gbad = []
        for kind, key in (("actor", "grads_actor"), ("critic", "grads_critic")):
            for name, gref in stats[0][key].items():
                off, shape = offs[kind][name]
                gm = learner.first_grads[kind][a, off:off + gref.numel()].view(gref.shape).cpu()
                rel = float((gm - gref).abs().max() / (gref.abs().max() + 1e-12))
                gbad.append((rel, kind + ":" + name, float(gref.abs().max())))
        gbad.sort(reverse=True)
        worst_grad = max(worst_grad, gbad[0][0])
        print(f"[learner highway-shape a={a}] pre {dpre}\n   worst first-epoch grads (rel, name, |ref|max): {gbad[:4]}")
        for kind, nets, ref in (("actor", mac.agents, ap), ("critic", mac.critics, cp)):
            sd = nets[a].state_dict()
            for k, v in ref.items():
                d = (sd[k].detach().cpu().double() - v.double()).abs()
                n_off += int((d > 5e-5).sum())
                n_all += d.numel()
                if d.numel() and float(d.max()) > 2e-5:
                    print(f"   a={a} {kind}:{k} max diff {float(d.max()):.3e} at {int(d.argmax())} "
                          f"n(>2e-5)={int((d > 2e-5).sum())} of {d.numel()}")
                worst = max(worst, maxdiff(sd[k], v))
    print(f"[learner highway-shape] worst post-train weight diff vs oracle {worst:.3e}; "
          f"worst first-epoch gradient rel diff {worst_grad:.3e}; weights off by >5e-5: {n_off} of {n_all}")
    # Well-conditioned check: every first-epoch gradient tensor agrees to 1e-5 of its scale.
    assert worst_grad < 1e-5
    # After 3 Adam steps the weights agree to 5e-5 except where a ReLU pre-activation of ONE
    # (row, unit) sits within fp32 noise of zero: the two implementations then disagree on that
    # unit's mask and, with only 99 training rows, one net's weights move by up to ~lr.  That is
    # a property of ReLU + fp32 (the reference vs its own GPU build shows the same), so allow a
    # small fraction of such weights but bound them by a few learning rates.
    assert worst < 4 * args.lr and n_off < 0.01 * n_all


@pytest.mark.parametrize("shape", [(2, 300, 272), (1, 128, 2485), (3, 1000, 2485)])
def test_fc1_matches_fp64(shape):
    """The fc1 forward and backward tensor-core products (csrc/fc1_mma.cu) against an fp64 reference on the same operands:
    ragged rows, ragged K (Fp = 288 is not a multiple of the 64-wide k-block)."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "check_fc1", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "check_fc1.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.run(*shape, reps=1) < 1e-5


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_prediction_learn_vs_reference_golden(case):
    """SURVEY §8f rank 2 — Prediction_policy.learn (csrc/pred_learn.cu: GAT + decoder forward, masked L1, full backward,
    clip, Adam) against one recorded call of the reference's ``learn`` (same sampled transitions, Gumbel noise and
    dropout masks): loss, every gradient tensor vs the oracle's autograd, post-step weights vs the reference."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "check_pred_learn", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "check_pred_learn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.run(case)


@pytest.mark.parametrize("case", ["mpe", "highway"])
def test_behavior_learn_vs_reference_golden(case):
    """SURVEY §8f rank 3 — Behavior_policy.learn (csrc/beh_learn.cu: decoder / encoder GRUs over every window position,
    latent recursion, one BPTT, clip, Adam) against one recorded call of the reference's ``learn`` (same dropout masks):
    losses, every gradient tensor vs the oracle, post-step weights vs the reference."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib
    mod = importlib.import_module("tools.check_beh_learn")
    assert mod.run(case)


def test_behavior_learn_tiled_kernels_match_the_draft_on_ragged_tiles():
    """csrc/beh_learn_tile.cu (the default: 64-chain CTA tiles, three launches) against csrc/beh_learn.cu (one warp per
    chain, pinned to the reference by the test above) on the same inputs and dropout masks: 6 episodes x 55 slots = 330
    chains per agent-net = five full tiles and a ragged one, agents terminating inside the episode."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import importlib
    mod = importlib.import_module("tools.check_beh_learn_tile")
    assert mod.run(envs=6, steps=25)


def test_packed_batch_last_action_with_list_bs_and_popart_checkpoint_formats(tmp_path):
    """ADVICE round 1: (a) ``update(..., bs=[0, 2])`` (the pymarl ``envs_not_terminated`` pattern) must reach the packed
    rows' last-action columns; (b) critic checkpoints in the CUDA reference's format (no ``v_out.*`` keys, 20 optimiser
    parameters: utils/mappo_utils/popart.py:21-27 on CUDA) load, and ``popart_cuda_quirk`` writes that format."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.config import make_args
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from iplan_b200.learners.ippo_learner import IPPOLearner
    args = make_args("MPE", batch_size_run=3, buffer_size=3, batch_size=2, use_cuda=True, device="cuda")
    scheme, groups, pre = make_scheme(args)
    batch = EpisodeBatch(scheme, groups, 3, args.episode_limit + 1, preprocess=pre, device="cuda")
    d = batch.packed_dims
    acts = torch.tensor([[[1], [2], [3]], [[4], [0], [1]]])                     # [2 envs, A = 3, 1]
    batch.update({"actions": acts}, bs=[0, 2], ts=1, mark_filled=False)
    cols = batch.packed[:, :, 2, d.col_act:d.col_act + d.n_actions].cpu()       # row t + 1 holds onehot(a_t)
    assert cols[:, 0].argmax(-1).tolist() == [1, 2, 3] and cols[:, 2].argmax(-1).tolist() == [4, 0, 1]
    assert float(cols[:, 1].abs().sum()) == 0.0 and float(cols[:, 0].sum()) == 3.0
    # ---- checkpoint formats
    mac = DcntrlMAC(batch.scheme, groups, args)
    sd = {k: v.clone() for k, v in mac.critics[0].state_dict().items()}
    cuda_fmt = {k: v + 1.0 for k, v in sd.items() if not k.startswith("v_out.")}
    assert len(cuda_fmt) == 20 and len(sd) == 26
    keep = mac.critics[0].state_dict()["v_out.weight"].clone()
    mac.critics[0].load_state_dict(cuda_fmt)                                    # strict load of the 20-key format
    new = mac.critics[0].state_dict()
    assert torch.equal(new["v_out.weight"], keep) and torch.allclose(new["base.mlp.fc2.0.0.weight"], sd["base.mlp.fc2.0.0.weight"] + 1.0)
    with pytest.raises(RuntimeError):
        mac.critics[0].load_state_dict({k: v for k, v in sd.items() if k != "rnn.norm.bias"})       # other keys still strict
    args.popart_cuda_quirk = True
    mac2 = DcntrlMAC(batch.scheme, groups, args)
    learner = IPPOLearner(mac2, batch.scheme, Log(), args)
    learner.steps["critic"] = 3
    mac2.save_models(str(tmp_path))
    learner.save_models(str(tmp_path))
    assert not any(k.startswith("v_out.") for k in torch.load(tmp_path / "critic_0.th", weights_only=False))
    opt = torch.load(tmp_path / "critic_0_opt.th", weights_only=False)
    assert len(opt["param_groups"][0]["params"]) == 20
    assert float(learner.masks["critic"][mac2.critic_stack.named_offsets()["v_out.weight"][0]]) == 0.0
    learner.load_models([str(tmp_path)] * 3, load_optimisers=True)
