"""Time IPPOLearner.train at the benchmark's update shape for num_mini_batch = 1, 2, 4, 8, and the row gather alone:

    python tools/bench_minibatch.py [--envs 512] [--reps 3] [--k 1 2 4 8]

Highway, 5 agents, T = 90, buffer = envs, batch_size = envs - 1 (45 990 training rows at 512 envs), 15 epochs.  One
device-resident rollout supplies the episode batch; every timed call inserts that same batch and trains on it from the
weights the previous call left.  One warm-up train() per num_mini_batch, then the values alternate ``reps`` times; each
train() is timed with CUDA events around the call (it ends in the copy of the statistics to the host).  A separate,
untimed-in-total train() with 4 mini-batches records the learner's event timeline and gives the gather kernel's time
per mini-batch; its bytes are the f16 hi / lo operand rows it reads and writes (agents x rows x 2 x ldx x 2 B, each
way), set against the 3.35 TB/s of HBM3 the H100 SXM data sheet gives.  Prints the card's name and power limit with
the numbers, and one JSON line.  Needs a CUDA device."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_behavior_learn import card                              # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet; not a rate this card has been measured to reach


def gather_bytes(n_agents, rows, ldx):
    """Bytes one gather of ``rows`` rows per agent moves for the f16 hi / lo operand copies: read + write."""
    return 2 * n_agents * rows * 2 * ldx * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--k", type=int, nargs="+", default=[1, 2, 4, 8])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_minibatch needs a CUDA device")
    from iplan_b200.runners.synthetic_runner import build_system
    sysm = build_system(n_envs=a.envs, env="highway", hazard=0.01, seed=112358, batch_size=a.envs - 1)
    learner, args = sysm.learner, sysm.args
    batch, *_ = sysm.runner.run()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    gathered = {}                # the gathered copy of each num_mini_batch, kept so that alternating does not reallocate it

    def train(k):
        learner.num_mini_batch, learner.mb = k, gathered.get(k)
        learner.insert_episode_batch(batch)
        torch.cuda.synchronize()
        ev0.record()
        learner.train(0)
        ev1.record()
        ev1.synchronize()
        gathered[k] = learner.mb
        return ev0.elapsed_time(ev1)

    times = {k: [] for k in a.k}
    for it in range(a.reps + 1):                     # iteration 0 warms up every value
        for k in a.k:
            ms = train(k)
            if it > 0:
                times[k].append(ms)
    # the gather alone, from the learner's event timeline of one more update
    kg = 4
    learner.events = []
    train(kg)
    torch.cuda.synchronize()
    lev, learner.events = learner.events, None
    gather_ms = sorted(e.elapsed_time(lev[i + 1][1]) for i, (tag, e) in enumerate(lev[:-1]) if tag == "gather")
    n = args.batch_size * args.episode_limit
    ldx = learner.store["X"].shape[-1]
    nbytes = gather_bytes(args.n_agents, n // kg, ldx)
    g_med = gather_ms[len(gather_ms) // 2]
    rate = nbytes / (g_med * 1e-3)
    gpu, plim = card()
    med = {k: sorted(ts)[len(ts) // 2] for k, ts in times.items()}
    print(f"IPPOLearner.train on {gpu} (power limit {plim} W): {a.envs} episodes x T = {args.episode_limit}, {args.n_agents} agents, "
          f"ldx = {ldx}, {n} training rows, {args.ppo_epoch} epochs")
    for k, ts in times.items():
        print(f"  num_mini_batch {k}: median {med[k]:.1f} ms over {len(ts)} calls ({', '.join(f'{t:.1f}' for t in ts)}); "
              f"{args.ppo_epoch * k} Adam steps per net")
    print(f"  gather_rows ({kg} mini-batches of {n // kg} rows): median {g_med * 1e3:.0f} us of {len(gather_ms)} launches, "
          f"{nbytes / 1e6:.0f} MB read + written -> {rate / 1e12:.2f} TB/s = {100 * rate / HBM_BYTES_PER_S:.0f} % of the "
          f"{HBM_BYTES_PER_S / 1e12:.2f} TB/s data-sheet bandwidth; {args.ppo_epoch * kg * g_med:.1f} ms per train()")
    print(json.dumps(dict(gpu=gpu, power_limit_w=plim, envs=a.envs, rows=n, ldx=ldx, epochs=args.ppo_epoch, train_ms=times,
                          train_median_ms=med, gather_k=kg, gather_us_median=g_med * 1e3, gather_bytes=nbytes,
                          gather_bytes_per_s=rate)))


if __name__ == "__main__":
    main()
