"""Drop-in test (SURVEY §4 iii): the REFERENCE'S OWN ``ParallelRunner.run`` body
(oracle/_ref/runners/ippo_parallel_runner.py:105-281, staged unmodified by oracle/make_ref.py) drives the iplan_b200
objects — DcntrlMAC, Prediction_policy, Behavior_policy, EpisodeBatch (and, in one variant, the observation wrapper) —
swapped in exactly as INTEGRATION.md prescribes, and the episode it stores is compared with the one the same runner body
stores when it drives the reference's own objects on the CPU: same weights, same synthetic env, same Gumbel noise, same
sampled actions.  Tolerance 1e-4 (north_star)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOL = 1e-4


def _run_reference(R, B, T, seed):
    """The reference end to end on the CPU; records the Gumbel noise of every GAT_Net.forward and every
    select_actions_ippo result while its runner runs."""
    import torch.nn.functional as Fn
    args = R.ref_args("highway", batch_size_run=B, episode_limit=T, buffer_size=B, batch_size=B - 1)
    ref = R.build_reference(args, seed)
    with torch.no_grad():
        for ag in ref.mac.agents:                       # gain-0.01 init gives ~uniform logits: make the head non-degenerate
            ag.act.action_out.linear.weight.mul_(40.0)
            ag.act.action_out.linear.bias.uniform_(-0.5, 0.5)
            ag.base.feature_norm.weight.uniform_(0.5, 1.5)
            ag.base.feature_norm.bias.uniform_(-0.2, 0.2)
        for cr in ref.mac.critics:
            cr.base.feature_norm.weight.uniform_(0.5, 1.5)
            cr.base.feature_norm.bias.uniform_(-0.2, 0.2)
    runner = R.build_runner(ref, R.SyntheticHostEnv(args, B, hazard=0.05, seed=seed))
    gumbels, selects = [], []
    orig_gs = Fn.gumbel_softmax

    def recording_gumbel_softmax(logits, tau=1, hard=False, eps=1e-10, dim=-1):
        g = -torch.empty_like(logits).exponential_().log()          # torch.nn.functional.gumbel_softmax's own draw
        gumbels.append(g.detach().clone())
        return ((logits + g) / tau).softmax(dim)

    orig_sel = ref.mac.select_actions_ippo

    def recording_select(batch, t_ep, test_mode=False):
        out = orig_sel(batch, t_ep=t_ep, test_mode=test_mode)
        selects.append(dict(values=np.array(out[0]), actions=np.array(out[1]),
                            logp=torch.cat([l.reshape(-1, 1) for l in out[2]], dim=1).detach().clone(),
                            rnn_a=np.array(out[3]), rnn_c=np.array(out[4])))
        return out

    ref.mac.select_actions_ippo = recording_select
    Fn.gumbel_softmax = recording_gumbel_softmax
    try:
        torch.manual_seed(seed)
        with torch.no_grad():
            batch, *_ = runner.run(test_mode=False)
    finally:
        Fn.gumbel_softmax = orig_gs
    return args, ref, batch, gumbels, selects


@pytest.mark.parametrize("own_wrapper", [False, True])
def test_reference_runner_body_drives_iplan_b200_objects(own_wrapper):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from oracle import ref_driver as R
    if not R.available():
        pytest.skip("oracle/_ref not staged (python oracle/make_ref.py in the build container)")
    from iplan_b200.components.episode_buffer import EpisodeBatch
    from iplan_b200.controllers.dcntrl_controller import DcntrlMAC
    from iplan_b200.nova.prediction_policy import Prediction_policy
    from iplan_b200.nova.stable_behavior_policy import Behavior_policy
    from iplan_b200.observation_wrapper import observersation_state_history_wrapper as OwnWrapper

    B, T, seed = 3, 12, 5
    args, ref, ref_batch, gumbels, selects = _run_reference(R, B, T, seed)
    A, N = args.n_agents, args.max_vehicle_num
    n_gat = len(gumbels) // A
    assert len(gumbels) == A * n_gat and n_gat == T + 1 and len(selects) == T

    # ---- the same runner body with the iplan_b200 objects (INTEGRATION.md §1) ---------------------------------
    import runners.ippo_parallel_runner as ref_runner_mod                      # staged reference module
    import copy
    gargs = copy.copy(args)
    gargs.use_cuda, gargs.device, gargs.buffer_cpu_only = True, "cuda", False
    scheme, groups, preprocess = R.make_scheme(gargs)
    from iplan_b200.components.transforms import OneHot
    preprocess = {"actions": ("actions_onehot", [OneHot(out_dim=gargs.n_actions)])}
    proto = EpisodeBatch(scheme, groups, 1, 2, preprocess=preprocess, device="cuda")
    mac = DcntrlMAC(proto.scheme, groups, gargs)
    pred, beh = Prediction_policy(gargs, None), Behavior_policy(gargs, None)
    for i in range(A):
        mac.agents[i].load_state_dict(ref.mac.agents[i].state_dict())
        mac.critics[i].load_state_dict(ref.mac.critics[i].state_dict())
        pred.pred_GAT[i].load_state_dict(ref.prediction.pred_GAT[i].state_dict())
        beh.behavior_encoder[i].load_state_dict(ref.behavior.behavior_encoder[i].state_dict())

    # feed the recorded noise: call c of GAT_latent_update consumed gumbels[c*A : (c+1)*A] (one per agent-net, :101-113)
    calls = {"gat": 0, "sel": 0}
    orig_gat = pred.GAT_latent_update

    def gat_with_recorded_noise(history_single, encoder_hidden, behavior_latent=None):
        c = calls["gat"]
        pred.debug_gumbel = torch.stack([gumbels[c * A + i].view(B, N, N - 1, 2) for i in range(A)]).cuda().contiguous()
        calls["gat"] += 1
        return orig_gat(history_single, encoder_hidden, behavior_latent)

    pred.GAT_latent_update = gat_with_recorded_noise
    orig_sel = mac.select_actions_ippo
    mac.capture_logits = True
    sel_diffs = []

    def select_with_recorded_actions(batch, t_ep, test_mode=False):
        values, actions, logps, rnn_a, rnn_c = orig_sel(batch, t_ep=t_ep, test_mode=test_mode)
        rec = selects[calls["sel"]]
        calls["sel"] += 1
        # the sampled actions are the reference's; our distribution must give them the reference's log-probability
        logits = mac.last_logits.permute(1, 0, 2).float().cpu()                  # [B,A,n_actions]
        lp = torch.log_softmax(logits, dim=-1).gather(-1, torch.as_tensor(rec["actions"]).long().unsqueeze(-1)).squeeze(-1)
        sel_diffs.append((float(np.abs(values - rec["values"]).max()), float((lp - rec["logp"]).abs().max()),
                          float(np.abs(rnn_a - rec["rnn_a"]).max()), float(np.abs(rnn_c - rec["rnn_c"]).max())))
        assert rnn_a.shape == rec["rnn_a"].shape and values.shape == rec["values"].shape and actions.shape == rec["actions"].shape
        return values, rec["actions"], logps, rnn_a, rnn_c

    mac.select_actions_ippo = select_with_recorded_actions

    saved = (ref_runner_mod.EpisodeBatch, ref_runner_mod.observersation_state_history_wrapper)
    ref_runner_mod.EpisodeBatch = EpisodeBatch                                 # runners/ippo_parallel_runner.py:2
    if own_wrapper:
        ref_runner_mod.observersation_state_history_wrapper = OwnWrapper       # :4
    try:
        runner = ref_runner_mod.ParallelRunner(gargs, R.SyntheticHostEnv(gargs, B, hazard=0.05, seed=seed), R.NullLogger())
        runner.setup(scheme, groups, preprocess, mac, beh, pred)
        batch, *_ = runner.run(test_mode=False)
    finally:
        ref_runner_mod.EpisodeBatch, ref_runner_mod.observersation_state_history_wrapper = saved
    torch.cuda.synchronize()
    assert calls["gat"] == T + 1 and calls["sel"] == T
    assert getattr(batch, "packed", None) is not None, "the runner must have filled the packed device batch"

    worst = {}
    for key in ("history", "attention_latent", "behavior_latent", "rnn_states_actors", "rnn_states_critics", "reward"):
        d = float((batch[key].float().cpu() - ref_batch[key].float()).abs().max())
        worst[key] = d
    for key in ("actions", "terminated", "filled", "avail_actions"):
        assert torch.equal(batch[key].cpu().long(), ref_batch[key].long()), key
    assert torch.equal(batch["actions_onehot"].cpu().float(), ref_batch["actions_onehot"].float())
    dv, dlp, dra, drc = (max(x[i] for x in sel_diffs) for i in range(4))
    print(f"[drop-in own_wrapper={own_wrapper}] stored-episode diffs {worst}; select_actions: values {dv:.2e} logp {dlp:.2e} rnn {dra:.2e}/{drc:.2e}")
    assert worst["history"] < 1e-6 and worst["reward"] < 1e-6
    assert all(v < TOL for v in worst.values()), worst
    assert dv < TOL and dlp < TOL and dra < TOL and drc < TOL
