"""Time Behavior_policy.learn of the soft-update module (iPLAN), the hard-update module (iPLAN-Hard) and the
fully-connected module (iPLAN-FC) on the same batch, and the rollout step of the FC and soft encoders:

    python tools/bench_behavior_learn.py [--envs 512] [--steps 90] [--reps 3] [--rollout-envs 512]

Highway shape (5 agents x 55 slots, W = 10), Philox dropout.  One warm-up call of each, then the three alternate; each
call is timed with CUDA events around ``learn`` (kernels, gradient clipping, Adam and the copy of the losses to the
host).  The FC leg also reports FLOP/s against the multiply-adds its rows need (forward, input and weight gradients of
both networks).  The rollout leg runs one warm-up and one timed episode of the device runner per module and reports the
median of the runner's per-step "beh" events (the encoder step kernel).  Prints the card's name and power limit with
the times, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iplan_b200.config import make_args                                  # noqa: E402
from iplan_b200.nova import behavior_FC_policy, behavior_policy, stable_behavior_policy      # noqa: E402
from tools.check_beh_learn_tile import make_batch                        # noqa: E402


def card():
    """Name and power limit of the current device (read-only nvidia-smi query)."""
    idx = torch.cuda.current_device()
    name, plim = torch.cuda.get_device_name(idx), None
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        plim = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return name, plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=90)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rollout-envs", type=int, default=512)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_behavior_learn needs a CUDA device")
    args = make_args("highway", use_cuda=True, device="cuda")
    batch = make_batch(args, a.envs, a.steps + 1, seed=5)
    torch.manual_seed(0)
    pols = {"soft": stable_behavior_policy.Behavior_policy(args, None), "hard": behavior_policy.Behavior_policy(args, None),
            "fc": behavior_FC_policy.Behavior_policy(args, None)}
    times = {k: [] for k in pols}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(a.reps + 1):                     # iteration 0 warms up both
        for name, pol in pols.items():
            torch.cuda.synchronize()
            ev0.record()
            pol.learn(batch, t_env=0)
            ev1.record()
            ev1.synchronize()
            if it > 0:
                times[name].append(ev0.elapsed_time(ev1))
    gpu, plim = card()
    shape = f"{a.envs} envs x {a.steps} steps x {args.n_agents} agents x {args.max_vehicle_num} slots"
    print(f"Behavior_policy.learn on {gpu} (power limit {plim} W), {shape}:")
    for name, ts in times.items():
        print(f"  {name}: median {sorted(ts)[len(ts) // 2]:.1f} ms over {len(ts)} calls ({', '.join(f'{t:.1f}' for t in ts)})")
    flop = 2 * fc_macs(args, a.envs, a.steps)
    fc_ms = sorted(times["fc"])[len(times["fc"]) // 2]
    print(f"  fc: {flop / 1e12:.3f} TFLOP per call -> {flop / fc_ms / 1e9:.1f} TFLOP/s")
    step = rollout_step_ms(a.rollout_envs) if a.rollout_envs > 0 else {}
    for name, ms in step.items():
        print(f"  rollout encoder step ({name}, {a.rollout_envs} envs): median {ms * 1e3:.1f} us per step")
    print(json.dumps(dict(gpu=gpu, power_limit_w=plim, envs=a.envs, steps=a.steps, agents=args.n_agents, slots=args.max_vehicle_num,
                          soft_ms=times["soft"], hard_ms=times["hard"], fc_ms=times["fc"], fc_tflop=flop / 1e12,
                          rollout_envs=a.rollout_envs, rollout_beh_step_ms=step)))


def fc_macs(args, envs, steps):
    """Multiply-adds of one FC learn call: per row the forward of both networks, the decoder's input gradient (hidden
    layers and the latent columns), the encoder's input gradient (hidden layers) and every weight gradient."""
    K0, L, E, Dh = args.obs_shape_single * args.max_history_len, args.latent_dim, args.encoder_rnn_dim, args.decoder_rnn_dim
    rows = envs * args.max_vehicle_num * (steps - 1 - args.max_history_len) * args.n_agents
    enc = K0 * E + E * E + E * L
    dec = (K0 + L) * Dh + Dh * Dh + Dh * K0
    return rows * (2 * enc + 2 * dec + (Dh * K0 + Dh * Dh + Dh * L) + (E * L + E * E))


def rollout_step_ms(envs):
    """Median per-step time of the runner's "beh" events (the behaviour encoder's rollout kernel) for the FC and soft
    modules, one warm-up episode each."""
    from iplan_b200.runners.synthetic_runner import build_system
    out = {}
    for name, over in (("fc", dict(behavior_fully_connected=True)), ("soft", {})):
        sysm = build_system(n_envs=envs, env="highway", seed=3, **over)
        sysm.runner.run(test_mode=True)
        sysm.runner.gat_events = []
        sysm.runner.run(test_mode=True)
        torch.cuda.synchronize()
        ts = sorted(e0.elapsed_time(e1) for tag, e0, e1 in sysm.runner.gat_events if tag == "beh")
        sysm.runner.gat_events = None
        out[name] = ts[len(ts) // 2]
    return out


if __name__ == "__main__":
    main()
