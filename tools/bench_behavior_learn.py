"""Time Behavior_policy.learn of the soft-update module (iPLAN) and the hard-update module (iPLAN-Hard) on the same batch:

    python tools/bench_behavior_learn.py [--envs 512] [--steps 90] [--reps 3]

Highway shape (5 agents x 55 slots, W = 10), Philox dropout.  One warm-up call of each, then the two alternate; each call
is timed with CUDA events around ``learn`` (kernels, gradient clipping, Adam and the copy of the losses to the host).
Prints the card's name and power limit with the times, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from iplan_b200.config import make_args                                  # noqa: E402
from iplan_b200.nova import behavior_policy, stable_behavior_policy      # noqa: E402
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
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_behavior_learn needs a CUDA device")
    args = make_args("highway", use_cuda=True, device="cuda")
    batch = make_batch(args, a.envs, a.steps + 1, seed=5)
    torch.manual_seed(0)
    pols = {"soft": stable_behavior_policy.Behavior_policy(args, None), "hard": behavior_policy.Behavior_policy(args, None)}
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
    print(json.dumps(dict(gpu=gpu, power_limit_w=plim, envs=a.envs, steps=a.steps, agents=args.n_agents, slots=args.max_vehicle_num,
                          soft_ms=times["soft"], hard_ms=times["hard"])))


if __name__ == "__main__":
    main()
