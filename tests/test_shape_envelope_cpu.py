"""The shape envelope of every compute entry point, from the outside: each call below has exactly one size just past what
its kernel is built for, and must return a nonzero code with an iplan_last_error() text that names that size.  Every one
of these checks runs before the entry point's first CUDA call, so no device is needed and no pointer is ever followed
(the buffers are placeholder addresses).  The joint shared-memory limits are pinned through the header's
IPLAN_CTRL_MAX_FEAT and IPLAN_PRED_LEARN_MAX_SLOTS; that each is accepted is shown on the GPU
(tests/test_gpu_shape_envelope.py)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = C.c_void_p(0x1000)            # non-null, never dereferenced: every call below fails an argument check first


def _header_define(name):
    text = open(os.path.join(ROOT, "include", "iplan_b200.h")).read()
    return int(re.search(rf"#define {name} (\d+)", text).group(1))


def _lib():
    from iplan_b200 import _lib
    return _lib


def _rejects(rc, *needles):
    msg = _lib().lib.iplan_last_error().decode()
    assert rc != 0, f"accepted; last error {msg!r}"
    for n in needles:
        assert n in msg, (n, msg)
    return msg


def _view(dim):
    L = _lib()
    return L.View(0x1000, 64 * 64 * dim, 64 * dim, dim)


# ---- K1 --------------------------------------------------------------------------------------------------------------
def _gat_step(n_slots=6, obs_dim=4, latent_dim=8, n_envs=3):
    L = _lib()
    scratch = max(1, L.lib.iplan_gat_scratch_floats(n_envs, 2, max(n_slots, 2)))
    return L.lib.iplan_gat_step(FAKE, 1024, _view(obs_dim), _view(latent_dim), _view(32), _view(32), None, 1, 0, 1.0,
                                None, FAKE, scratch, n_envs, 2, n_slots, obs_dim, latent_dim, None)


@pytest.mark.parametrize("n_slots", [1, 0, 65])
def test_k1_rejects_slot_counts_outside_2_to_64(n_slots):
    _rejects(_gat_step(n_slots=n_slots), "gat_step", f"n_slots {n_slots} not in [2,64]")


@pytest.mark.parametrize("obs_dim,latent_dim", [(9, 8), (4, 13), (16, 1)])
def test_k1_rejects_input_width_17(obs_dim, latent_dim):
    _rejects(_gat_step(obs_dim=obs_dim, latent_dim=latent_dim), "gat_step", "obs_dim+latent_dim 17 > 16")


def test_k1_header_limit_is_the_checked_one():
    assert _header_define("IPLAN_MAX_SLOTS") == 64


# ---- K1b -------------------------------------------------------------------------------------------------------------
def _beh_step(obs_dim=5, latent_dim=8, hist_len=10, n_slots=7, win_stride=0, win_pad=0):
    L = _lib()
    return L.lib.iplan_behavior_step_ex(FAKE, 1024, _view(hist_len * obs_dim), win_stride, win_pad, _view(32),
                                        _view(latent_dim), _view(latent_dim), 0.5, 3, 2, n_slots, obs_dim, latent_dim,
                                        hist_len, None)


def test_k1b_rejects_obs_dim_8_like_the_behaviour_learner():
    _rejects(_beh_step(obs_dim=8, hist_len=8), "behavior_step", "obs_dim 8 not in [1,7]")
    _rejects(_beh_step(obs_dim=0, hist_len=8), "behavior_step", "obs_dim 0 not in [1,7]")


@pytest.mark.parametrize("obs_dim,hist_len", [(5, 13), (1, 65), (7, 10)])
def test_k1b_rejects_window_over_64_floats(obs_dim, hist_len):
    _rejects(_beh_step(obs_dim=obs_dim, hist_len=hist_len), "behavior_step", f"hist_len*obs_dim {obs_dim * hist_len} > 64")


@pytest.mark.parametrize("latent_dim", [0, 9])
def test_k1b_rejects_latent_dim_outside_1_to_8(latent_dim):
    _rejects(_beh_step(latent_dim=latent_dim), "behavior_step", f"latent_dim {latent_dim} not in [1,8]")


def test_k1b_rejects_a_pad_of_the_whole_window():
    _rejects(_beh_step(win_stride=5 * 55, win_pad=10), "behavior_step", "win_pad 10 not in [0,10)")


def test_k1b_plain_entry_point_checks_alike():
    L = _lib()
    rc = L.lib.iplan_behavior_step(FAKE, 1024, _view(64), _view(32), _view(8), _view(8), 0.5, 3, 2, 7, 8, 8, 8, None)
    _rejects(rc, "obs_dim 8 not in [1,7]")


# ---- K1c -------------------------------------------------------------------------------------------------------------
def _ctrl(feat_dim=37, n_actions=5):
    L = _lib()
    return L.lib.iplan_controller_step(FAKE, 4096, FAKE, 4096, FAKE, 4096, 4096, FAKE, FAKE, FAKE, FAKE, 64, 64, 64, 64,
                                       None, None, 1, 0, 0, FAKE, FAKE, FAKE, None, None, None,
                                       19, 2, feat_dim, n_actions, None)


@pytest.mark.parametrize("n_actions", [0, 9, -1])
def test_k1c_rejects_action_counts_outside_1_to_8(n_actions):
    _rejects(_ctrl(n_actions=n_actions), "controller_step", f"n_actions {n_actions} not in [1,8]")


def test_k1c_rejects_one_feature_past_its_shared_memory():
    top = _header_define("IPLAN_CTRL_MAX_FEAT")
    assert top == 2800
    _rejects(_ctrl(feat_dim=top + 1), "controller_step", f"feat_dim {top + 1} needs", "shared memory")


def test_k1c_rejects_the_highway_width_at_63_slots():
    """Highway widths (obs_dim 5, attention 32, latent 8, 5 actions, 5 agents) at N = 63: feat_dim 2845.  K1 accepts
    63 slots; the controller does not, so the whole rollout stops at N = 62 (feat_dim 2800)."""
    from iplan_b200.config import controller_input_dim, make_args
    args = make_args("highway", n_other_vehicles=58)
    assert args.max_vehicle_num == 63
    F = controller_input_dim(args)
    assert F == 2845
    _rejects(_ctrl(feat_dim=F), "controller_step", "feat_dim 2845 needs", "shared memory")
    args62 = make_args("highway", n_other_vehicles=57)
    assert controller_input_dim(args62) == _header_define("IPLAN_CTRL_MAX_FEAT")


# ---- Prediction_policy.learn -----------------------------------------------------------------------------------------
def _pred_learn(n_slots=7, obs_dim=5, latent_dim=8, pred_len=5, scratch_floats=None):
    L = _lib()
    A, P = 2, 3
    if scratch_floats is None:
        scratch_floats = L.lib.iplan_pred_learn_scratch_floats(A, P, max(n_slots, 2), obs_dim, pred_len)
    return L.lib.iplan_pred_learn(FAKE, 4096, FAKE, 4096, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, FAKE, FAKE,
                                  FAKE, scratch_floats, 1, 0, 1.0, 0.1, A, P, n_slots, obs_dim, latent_dim, pred_len, None)


@pytest.mark.parametrize("n_slots,obs_dim,latent_dim", [(1, 5, 8), (65, 5, 8), (7, 9, 8), (7, 5, 12)])
def test_pred_learn_rejects_sizes_outside_its_kernel(n_slots, obs_dim, latent_dim):
    _rejects(_pred_learn(n_slots=n_slots, obs_dim=obs_dim, latent_dim=latent_dim), "pred_learn: bad sizes")


def test_pred_learn_rejects_one_slot_past_its_shared_memory():
    top = _header_define("IPLAN_PRED_LEARN_MAX_SLOTS")
    assert top == 57
    _rejects(_pred_learn(n_slots=top + 1), "pred_learn", f"n_slots {top + 1} needs", "shared memory")
    _rejects(_pred_learn(n_slots=64), "pred_learn", "n_slots 64 needs", "shared memory")


def test_pred_learn_rejects_a_short_scratch_before_launching():
    _rejects(_pred_learn(scratch_floats=10), "pred_learn: scratch too small")


# ---- Behavior_policy.learn -------------------------------------------------------------------------------------------
def _beh_windows(obs_dim=5, latent_dim=8, W=10, n_pos=8, win_step=10, win_first=0, T=90):
    L = _lib()
    A, B, N = 2, 3, 7
    scratch = L.lib.iplan_beh_learn_tile_scratch_floats(A, B, max(n_pos, 1), N, obs_dim, max(latent_dim, 1), W)
    return L.lib.iplan_beh_learn_windows(FAKE, 4096, FAKE, 4096, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE,
                                         scratch, 1, 0, 0.1, 1.0, 0.01, A, B, T, N, obs_dim, latent_dim, W, n_pos,
                                         win_step, win_first, None)


def test_behaviour_learner_rejects_obs_dim_8_like_k1b():
    _rejects(_beh_windows(obs_dim=8), "beh_learn", "obs_dim 8 not in [1,7]")
    _rejects(_beh_windows(obs_dim=0), "beh_learn", "obs_dim 0 not in [1,7]")


@pytest.mark.parametrize("latent_dim", [3, 7, 1, 10, 0])
def test_behaviour_learner_rejects_odd_or_wide_latents(latent_dim):
    _rejects(_beh_windows(latent_dim=latent_dim), "beh_learn", f"even latent_dim <= 8 is built (got {latent_dim})")


def test_behaviour_learner_rejects_targets_past_the_episode():
    _rejects(_beh_windows(n_pos=9), "beh_learn_windows", "target rows [10, 99] outside the episode of 90 steps")
    _rejects(_beh_windows(win_first=-11, n_pos=1), "beh_learn_windows", "outside the episode")
    _rejects(_beh_windows(win_step=0), "beh_learn_windows", "win_step >= 1")


def test_soft_behaviour_learner_checks_alike():
    L = _lib()
    scratch = L.lib.iplan_beh_learn_tile_scratch_floats(2, 3, 79, 7, 8, 8, 10)
    prev = L.lib.iplan_beh_learn_set_impl(0)
    try:
        rc = L.lib.iplan_beh_learn(FAKE, 4096, FAKE, 4096, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, scratch,
                                   1, 0, 0.1, 0.5, 0.01, 2, 3, 90, 7, 8, 8, 10, None)
    finally:
        L.lib.iplan_beh_learn_set_impl(prev)
    _rejects(rc, "beh_learn", "obs_dim 8 not in [1,7]")


# ---- IPPO learner tail -----------------------------------------------------------------------------------------------
def _tail(n_actions, feat_dim=316):
    L = _lib()
    ctx = L.LearnerCtx()
    for name in ("actor", "critic", "g_actor", "g_critic", "rnn_a", "rnn_c", "actions", "Z1", "A1", "Z2", "A2", "GI", "GH",
                 "stat", "SM", "old_logp", "old_value", "returns", "adv_raw", "alive", "norm", "stats"):
        setattr(ctx, name, 0x1000)
    ctx.actor_stride = ctx.critic_stride = 1 << 20
    ctx.feat_dim, ctx.n_actions, ctx.n_agents, ctx.T1, ctx.n_eps, ctx.n_train_eps = feat_dim, n_actions, 3, 11, 4, 4
    ctx.rnn_stride_agent, ctx.rnn_ld = 64 * 44, 64
    ctx.clip, ctx.ent_coef, ctx.v_coef, ctx.huber_delta, ctx.grad_scale = 0.2, 0.01, 1.0, 10.0, 1.0
    return L.lib.iplan_learner_tail(C.byref(ctx), 1, None)


@pytest.mark.parametrize("n_actions", [0, 9])
def test_learner_tail_rejects_action_counts_outside_1_to_8(n_actions):
    _rejects(_tail(n_actions), "learner_tail", f"n_actions {n_actions} not in [1,8]")
