#!/usr/bin/env python
"""bench.py — env-steps/sec of the iPLAN rollout-and-learn hot path on H100.

One "step" = one pass of the hot path over one batch of synthetic input: a 90-timestep
rollout of `envs_per_gpu` environments x 5 agents (K1 GAT + K1b behaviour encoder + K1c
controller per timestep) followed by one IPPOLearner.train (GAE, 15 PPO epochs, all agents).
Workload = BASELINE.json configs[2] "Hetero-Highway chaotic, 5 agents, 512 envs" per GPU
(weak scaling: every rank owns 512 envs; at N GPUs the job is 512*N envs, one NCCL
all-reduce of the actor+critic gradients per PPO epoch).

    python bench.py --gpus 1 --steps 3 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...
    python bench.py --impl reference ...      # the CPU port of the reference path, host cores

Prints ONE JSON line (rank 0).  `value` = device-resident path, inputs already in HBM;
`e2e` = the same work through the reference-facing numpy API (host buffers in/out every
timestep); `roofline` = the dominant kernel (K1 GAT step) timed with CUDA events inside the
timed region; `cpu_baseline` = the oracle port on the host cores (N=1 only).
`--dump-outputs DIR` writes what the last timed step computed as DIR/<name>.npy (float32; arrays larger than
DUMP_SAMPLE elements as a fixed, seeded sample of their elements), so that two builds can be compared output for output.
The inputs are the same in every run with the same arguments, and so are the outputs: the update's cross-block gradient
sums are added in a fixed order.  (--with-aux adds Behavior_policy.learn and Prediction_policy.learn, whose gradient sums
still use float atomics: with it the weights agree from run to run only to rounding.)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "env-steps/sec iPLAN Hetero-Highway chaotic (rollout + IPPO update)"


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", default="b200", choices=["b200", "reference"])
    p.add_argument("--envs-per-gpu", type=int, default=512)
    p.add_argument("--e2e-steps", type=int, default=3)
    p.add_argument("--no-cpu-baseline", action="store_true")
    p.add_argument("--no-e2e", action="store_true")
    p.add_argument("--workload", default="highway", choices=["highway", "microbench"],
                   help="highway = BASELINE configs[2] (headline); microbench = configs[4], the 8192 x 32 x 16 x 128-d GAT + GRU forward")
    p.add_argument("--with-aux", action="store_true",
                   help="also run Behavior_policy.learn and Prediction_policy.learn in every step (run_ippo.py:263-286 order) and report their time")
    p.add_argument("--dump-outputs", metavar="DIR", default=None,
                   help="after the timed steps, write the outputs of the last one as DIR/<name>.npy (rank 0)")
    return p.parse_args()


DUMP_SAMPLE = 1 << 20        # elements kept per dumped array (4 MB in float32)


def dump_outputs(out_dir, arrays):
    """arrays: name -> tensor.  Each is written flattened as float32; one with more than DUMP_SAMPLE elements is replaced by
    the elements at DUMP_SAMPLE sorted indices drawn with a fixed seed (the same indices for the same shape)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        t = t.detach().reshape(-1)
        if t.numel() > DUMP_SAMPLE:
            g = torch.Generator().manual_seed(20240601)
            idx = torch.randint(0, t.numel(), (DUMP_SAMPLE,), generator=g).sort().values
            t = t[idx.to(t.device)]
        np.save(os.path.join(out_dir, name + ".npy"), t.float().cpu().numpy())


def peaks():
    """NVIDIA's H100 SXM data-sheet figures (dense BF16 tensor rate, HBM3 bandwidth) at a 700 W limit: the yardstick of the
    roofline fractions, not rates this card has been measured to reach (a lower power limit lowers the attainable clocks)."""
    return dict(hbm=3350.0, tf_sus=989.0, src="H100 SXM data sheet, dense BF16")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region, and the card's name and power limit (read-only queries)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap,power.limit,name")

    def __init__(self, gpu_index):
        self.path = tempfile.mktemp(suffix=".csv")
        self.gpu = gpu_index
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, plim, name = [], [], set(), None, None
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in open(self.path):
            f = [x.strip() for x in line.split(",")]
            if len(f) < 10:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
                plim, name = float(f[8]), f[9]
            except ValueError:
                continue
            for n, v in zip(names, f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        os.unlink(self.path)
        sm.sort()
        return {"gpu": name, "power_limit_w": plim, "sm_mhz": sm[len(sm) // 2] if sm else None,
                "sm_max_mhz": max(mx) if mx else None, "samples": len(sm), "reasons": sorted(reasons)}


def gat_algorithmic(B, A, N, o, L, H=32):
    """Algorithmic FLOPs and HBM bytes of ONE K1 step, split over its two kernels:
    {"recur": (flops, bytes), "attend": (flops, bytes), "step": (flops, bytes)}.  Each node's inputs are counted
    once per kernel that needs them; the kernel-to-kernel logit scratch is not algorithmic traffic."""
    in_dim = o + L
    nodes = B * A * N
    recur = (2 * H * in_dim                     # encode
             + 2 * 2 * 2 * 3 * H * H            # factored input projections P, Q x 2 directions
             + 2 * (N - 1) * 2 * 3 * H * H      # bidirectional GRU recurrence
             + 2 * (N - 1) * 2 * 2 * H)         # hard-attention logits
    attend = (3 * 2 * H * H                     # q, k, v
              + (N - 1) * 2 * H * 2             # scores + weighted sum
              + 2 * 2 * 3 * H * H)              # GRUCell
    return {"recur": (recur * nodes, nodes * in_dim * 4),
            "attend": (attend * nodes, nodes * (in_dim + 2 * H) * 4),
            "step": ((recur + attend) * nodes, nodes * (in_dim + 2 * H) * 4)}


def run_reference(args):
    """--impl reference: the reference's OWN CPU implementation of the path (oracle/_ref, staged unmodified by
    oracle/make_ref.py) on the host cores; every step is the same FIXED sample (one full rollout timestep at 512 envs
    inside the reference's ParallelRunner.run + one IPPOLearner.train at Bf=64), extrapolated to the step.  Falls back
    to the oracle port (kind "port") only if oracle/_ref was not staged."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import torch
    from oracle import ref_driver as R
    Bl = args.envs_per_gpu
    T = 90
    if R.available():
        cores = R.usable_cpus()
        torch.set_num_threads(cores)
        runs, t_begin, budget_s = [], time.perf_counter(), 420.0
        for it in range(args.warmup + args.steps):
            # every step is the same fixed sample; once the wall budget is spent the remaining steps reuse the mean of
            # the samples already timed (steps_measured says how many were)
            if runs and time.perf_counter() - t_begin > budget_s:
                break
            m = R.measure(B=Bl, T=T, threads=cores, seed=it)
            if it >= min(args.warmup, 1):
                runs.append(m)
        t_step = sum(m["t_step"] for m in runs) / len(runs)
        t_train = sum(m["t_train"] for m in runs) / len(runs)
        kind, sample, sample_s = "reference", runs[-1]["sample"], sum(m["sample_s"] for m in runs) / len(runs)
        n_agents, slots = 5, 55
    else:
        from iplan_b200.config import make_args
        from oracle import cpu_baseline as cb
        a = make_args("highway", use_cuda=False, device="cpu")
        cores = cb.usable_cpus()
        torch.set_num_threads(cores)
        params = cb.random_params(a)
        times = []
        for it in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            ts = cb.time_rollout_steps(a, params, 128, 1, warmup=0, seed=it) * (Bl / 128)
            tt = cb.time_train(a, params, 8, seed=it) * (Bl / 8)
            if it >= args.warmup:
                times.append((ts, tt, time.perf_counter() - t0))
        t_step = sum(t[0] for t in times) / len(times)
        t_train = sum(t[1] for t in times) / len(times)
        kind, sample_s = "port", sum(t[2] for t in times) / len(times)
        sample = "oracle port (oracle/_ref not staged): 1 timestep at 128 envs x4, update at Bf=8 x64 in rows"
        n_agents, slots = a.n_agents, a.max_vehicle_num
    B = Bl * args.gpus
    # the CPU path does not shard: N x 512 envs cost N x the 512-env time
    step_s = (T * t_step + t_train) * args.gpus
    value = B * T / step_s
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_s * 1e3, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "Hetero-Highway chaotic, 5 agents, 512 envs/GPU, T=90, 15 PPO epochs (BASELINE configs[2])",
                   "envs": B, "envs_per_gpu": Bl, "agents": n_agents, "slots": slots, "feat_dim": 2485, "episode_limit": T,
                   "ppo_epoch": 15},
        "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": cores, "kind": kind, "sample": sample,
                         "t_rollout_step_s": t_step, "t_update_s": t_train},
        "extrapolation": {"measured_s_per_step": sample_s, "steps_measured": len(runs) if R.available() else args.steps,
                          "step_s": f"{T} x t_rollout_step_s + t_update_s" + (f", x{args.gpus} (no sharding on CPU)" if args.gpus > 1 else ""),
                          "note": "ms_per_step is the extrapolated full step (a full 512-env step of the reference takes ~10 min); "
                                  "the timed sample per step is fixed, not probe-sized"},
        "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


def log(msg):
    print(f"[bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


MB_ENVS, MB_AGENTS, MB_SLOTS, MB_DIM = 8192, 32, 16, 128
MB_METRIC = "env-steps/sec synthetic GAT+GRU microbench (8192 envs x 32 agent-nets x 16 slots x 128-d)"


def run_microbench_reference(args):
    """--impl reference --workload microbench: the reference's own GAT_Net at width 128 on the host cores, bounded sample."""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    import torch
    from oracle import ref_driver as R
    cores = R.usable_cpus()
    torch.set_num_threads(cores)
    per_item = []
    for it in range(args.warmup + args.steps):
        t = R.time_gat_net_128(n_envs=16, n_nets=2, seed=it)
        if it >= min(args.warmup, 1):
            per_item.append(t)
    t_item = sum(per_item) / len(per_item)
    step_s = t_item * MB_ENVS * MB_AGENTS                 # one forward of the whole 8192 x 32 problem (no sharding on CPU)
    value = MB_ENVS / step_s
    print(json.dumps({
        "impl": "reference", "metric": MB_METRIC, "value": value, "unit": "env-steps/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": step_s * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": "GAT_Net.forward, hidden 128, 16 slots, 8192 envs x 32 agent-nets (BASELINE configs[4])"},
        "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": cores, "kind": "reference",
                         "sample": f"the reference's own GAT_Net(128) (oracle/_ref) on 2 nets x 16 envs per step, scaled x{MB_ENVS * MB_AGENTS / 32:g} in items; {cores} torch threads"},
        "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


def run_microbench(args):
    """BASELINE configs[4]: one step = one GAT_Net.forward (width 128) over this rank's shard of the 8192 envs x 32 agent-nets."""
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from iplan_b200 import _lib
    from iplan_b200.nova.gat128 import GAT128
    envs = MB_ENVS // world                               # strong scaling: the 8192 envs are sharded, no exchange (forward only)
    A, N, H = MB_AGENTS, MB_SLOTS, MB_DIM
    net = GAT128(A, seed=0)                               # same weights on every rank (same seed)
    g = torch.Generator(device="cuda").manual_seed(112358 + rank)
    x = (torch.rand(A, envs, N, H, device="cuda", generator=g) * 2 - 1)
    h = torch.tanh(torch.randn(A, envs, N, H, device="cuda", generator=g))
    out = torch.empty_like(x)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        net.forward(x, h, out=out)
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = _lib.launch_count()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for k in range(args.steps):
        net.forward(x, h, out=out, events=evs[k])          # x (2.1 GB / rank at N=1) exceeds L2: nothing stays cached between steps
    e1.record()
    barrier()
    t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_per_step = float(t) / args.steps
    launches = (_lib.launch_count() - l0) / args.steps
    clocks = sampler.stop() if rank == 0 else None
    rec_ms = sum(a.elapsed_time(b) for a, b in evs) / args.steps
    # e2e: host buffers in, host result out, every step
    xh, hh = torch.empty(x.shape, pin_memory=True).copy_(x), torch.empty(h.shape, pin_memory=True).copy_(h)
    oh = torch.empty(x.shape, pin_memory=True)
    e2e_steps = max(1, min(args.steps, 3))
    barrier()
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        x.copy_(xh, non_blocking=True); h.copy_(hh, non_blocking=True)
        net.forward(x, h, out=out)
        oh.copy_(out, non_blocking=True)
        torch.cuda.synchronize()
    barrier()
    dt = torch.tensor([(time.perf_counter() - t0) / e2e_steps], device="cuda")
    if world > 1:
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    pk = peaks()
    f_recur, f_all, b_all = GAT128.algorithmic(A, envs)
    ach = f_recur / (rec_ms * 1e-3) / 1e12
    out_json = {
        "metric": MB_METRIC, "value": MB_ENVS / (ms_per_step / 1e3), "unit": "env-steps/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": "GAT_Net.forward, hidden 128, 16 slots, 8192 envs x 32 agent-nets (BASELINE configs[4])",
                   "envs": MB_ENVS, "envs_per_gpu": envs, "agent_nets": A, "slots": N, "dim": H,
                   "parallelism": f"env-sharded x{world} (forward only: no collective)", "l2": "inputs (2.1 GB per tensor per GPU at N=1) exceed L2"},
        "gpu_launches": launches, "library_gemms_per_step": 9, "clocks": clocks,
        "roofline": {"kernel": "gat128_recur_kernel (bidirectional 15-step GRU of every ego, W_hh in shared memory, wgmma m64n16k16 f16 x3 passes)",
                     "bound": "tensor", "achieved": ach, "peak": pk["tf_sus"], "unit": "TFLOP/s", "frac": ach / pk["tf_sus"], "traffic": None,
                     "peak_source": pk["src"], "launch_ms": rec_ms,
                     "algorithmic_flops_per_launch": f_recur, "share_of_step": rec_ms / ms_per_step,
                     "whole_op": {"algorithmic_flops": f_all, "algorithmic_bytes": b_all, "tflops": f_all / (ms_per_step * 1e-3) / 1e12,
                                  "hbm_frac_of_algorithmic_bytes": b_all / (ms_per_step * 1e-3) / 1e9 / pk["hbm"]}},
        "e2e": {"value": MB_ENVS / float(dt), "unit": "env-steps/s", "h2d_bytes_per_step": 2 * x.numel() * 4, "d2h_bytes_per_step": x.numel() * 4,
                "ms_per_step": float(dt) * 1e3, "steps": e2e_steps},
    }
    if world == 1 and not args.no_cpu_baseline:
        from oracle import ref_driver as R
        if R.available():
            torch.set_num_threads(R.usable_cpus())
            t_item = R.time_gat_net_128(n_envs=16, n_nets=2)
            v = MB_ENVS / (t_item * MB_ENVS * MB_AGENTS)
            out_json["cpu_baseline"] = {"value": v, "unit": "env-steps/s", "cores": R.usable_cpus(), "kind": "reference",
                                        "sample": "the reference's own GAT_Net(128) (oracle/_ref) on 2 nets x 16 envs, scaled in items"}
    print(json.dumps(out_json))
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"gat128_out": out})
    if world > 1:
        dist.destroy_process_group()


def main():
    args = parse()
    if args.workload == "microbench":
        return run_microbench_reference(args) if args.impl == "reference" else run_microbench(args)
    if args.impl == "reference":
        return run_reference(args)
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from iplan_b200 import _lib
    from iplan_b200.runners.synthetic_runner import build_system
    Bl = args.envs_per_gpu
    sysm = build_system(n_envs=Bl, env="highway", hazard=0.01, seed=112358 + rank,
                        batch_size=Bl * world - 1)          # global "first batch_size episodes" rule
    if world > 1:   # replicas start from identical weights (rank 0's)
        for t in (sysm.mac.actor_stack.flat, sysm.mac.critic_stack.flat, sysm.prediction.stack.flat, sysm.behavior.stack.flat):
            dist.broadcast(t, 0)
    a = sysm.args
    T = a.episode_limit

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    log(f"rank {rank}/{world}: system built, warm-up x{args.warmup}")
    for _ in range(args.warmup):
        sysm.run_and_train()
    barrier()
    log("timed region")
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    gat_events = []
    sysm.runner.gat_events = gat_events
    sysm.learner.events = []
    l0 = _lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    em = torch.cuda.Event(enable_timing=True)
    roll_ms = 0.0
    barrier()
    e0.record()
    for k in range(args.steps):
        s0 = torch.cuda.Event(enable_timing=True); s1 = torch.cuda.Event(enable_timing=True)
        s0.record()
        batch, *_ = sysm.runner.run()
        s1.record()
        sysm.learner.insert_episode_batch(batch)
        if args.with_aux:                                   # run_ippo.py:269-284: both auxiliary learners, then the IPPO update
            x0, x1, x2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            x0.record()
            sysm.behavior.learn(batch, sysm.runner.t_env)
            x1.record()
            sysm.prediction.learn(batch, sysm.runner.t_env)
            x2.record()
            gat_events.append(("aux_behavior_learn", x0, x1))
            gat_events.append(("aux_prediction_learn", x1, x2))
        sysm.learner.train(sysm.runner.t_env)
        gat_events.append(("roll", s0, s1))
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    launches = (_lib.launch_count() - l0) / args.steps
    clocks = sampler.stop() if rank == 0 else None
    sysm.runner.gat_events = None
    upd = {}
    lev = sysm.learner.events
    sysm.learner.events = None
    for (tag, e0), (_, e1) in zip(lev[:-1], lev[1:]):
        if tag != "end":
            upd[tag] = upd.get(tag, 0.0) + e0.elapsed_time(e1) / args.steps
    t = torch.tensor([ms], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
    ms_per_step = ms / args.steps
    value = Bl * world * T / (ms_per_step / 1e3)
    def times(tag):
        return [s.elapsed_time(e) for tg, s, e in gat_events if tg == tag]

    gat_ms, rec_ms, att_ms = times("gat"), times("gat_recur"), times("gat_attend")
    roll_ms = times("roll")
    gat_mean = sum(gat_ms) / max(1, len(gat_ms))
    rec_mean = sum(rec_ms) / max(1, len(rec_ms))
    breakdown = {tag: sum(times(tag)) / args.steps for tag in ("gat", "gat_recur", "gat_attend", "ctrl", "beh")}
    aux = {tag: sum(times(tag)) / args.steps for tag in ("aux_behavior_learn", "aux_prediction_learn")} if args.with_aux else None

    if rank == 0 and args.dump_outputs:
        # the last timed step: the episode its rollout stored and the weights its update produced.  Taken here, before the
        # e2e leg below runs more steps on the same system.
        dump = {k: batch[k] for k in ("actions", "reward", "terminated", "attention_latent", "behavior_latent")}
        dump.update(logp=sysm.runner.last_logp, values=sysm.runner.last_values,
                    actor_params=sysm.mac.actor_stack.flat, critic_params=sysm.mac.critic_stack.flat)
        if args.with_aux:
            dump.update(prediction_params=sysm.prediction.stack.flat, behavior_params=sysm.behavior.stack.flat)
        dump_outputs(args.dump_outputs, dump)

    # ---- e2e: same work through the reference-facing numpy API -----------------------------
    log(f"timed region done: {ms_per_step:.1f} ms/step; e2e leg")
    e2e = None
    if not args.no_e2e:
        sysm.run_and_train(api=True)                        # warm-up of the API path
        _lib.io_bytes["h2d"] = _lib.io_bytes["d2h"] = _lib.io_bytes["h2d_saved"] = 0
        barrier()
        t0 = time.perf_counter()
        for _ in range(args.e2e_steps):
            sysm.run_and_train(api=True)
        barrier()
        dt = torch.tensor([(time.perf_counter() - t0) / args.e2e_steps], device="cuda")
        if world > 1:
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        e2e = {"value": Bl * world * T / float(dt), "unit": "env-steps/s",
               "h2d_bytes_per_step": _lib.io_bytes["h2d"] // args.e2e_steps,
               "d2h_bytes_per_step": _lib.io_bytes["d2h"] // args.e2e_steps,
               "h2d_bytes_not_reuploaded_per_step": _lib.io_bytes["h2d_saved"] // args.e2e_steps,
               "ms_per_step": float(dt) * 1e3, "steps": args.e2e_steps,
               "path": "GAT_latent_update/latent_update/EpisodeBatch.update/select_actions_ippo with numpy buffers every timestep"}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    pk = peaks()
    alg = gat_algorithmic(Bl, a.n_agents, a.max_vehicle_num, a.obs_shape_single, a.latent_dim)
    att_mean = sum(att_ms) / max(1, len(att_ms))
    kname = "gat_recur_kernel (K1: encode, input projections, 2N GRU chains x N-1 steps, hard-attention logits; mma.sync)"
    flops, hbm_bytes = alg["recur"]
    k_ms, k_all = rec_mean, rec_ms
    ach_tf = flops / (k_ms * 1e-3) / 1e12 if k_ms > 0 else 0.0
    step_tf = alg["step"][0] / (gat_mean * 1e-3) / 1e12 if gat_mean > 0 else 0.0
    roofline = {"kernel": kname,
                "bound": "tensor", "achieved": ach_tf, "peak": pk["tf_sus"],
                "unit": "TFLOP/s", "frac": ach_tf / pk["tf_sus"],
                "peak_source": pk["src"],
                "launch_ms": k_ms, "launches_timed": len(k_all),
                "algorithmic_flops_per_launch": flops, "algorithmic_bytes_per_launch": hbm_bytes,
                "hbm_achieved_gbs": hbm_bytes / (k_ms * 1e-3) / 1e9 if k_ms > 0 else 0.0,
                "hbm_frac": (hbm_bytes / (k_ms * 1e-3) / 1e9) / pk["hbm"] if k_ms > 0 else 0.0,
                "share_of_step": sum(k_all) / ms if ms > 0 else None,
                "k1_step": {"launch_ms": gat_mean, "attend_ms": att_mean, "tflops": step_tf,
                            "algorithmic_flops": alg["step"][0], "algorithmic_bytes": alg["step"][1],
                            "share_of_step": sum(gat_ms) / ms if ms > 0 else None},
                "note": "fp32-accurate products cost 3 f16 MMAs each (hi/lo split): the tensor pipe does 3x the algorithmic FLOPs.  The "
                        "recurrence is a serial chain of N-1 steps per direction with its gate math between the products"}
    out = {
        "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": {"workload": "Hetero-Highway chaotic, 5 agents, 512 envs/GPU, T=90, 15 PPO epochs (BASELINE configs[2])",
                   "envs": Bl * world, "envs_per_gpu": Bl, "agents": a.n_agents, "slots": a.max_vehicle_num,
                   "feat_dim": sysm.mac.input_shape, "episode_limit": T, "ppo_epoch": a.ppo_epoch,
                   "parallelism": f"env-sharded x{world}", "l2": "inputs (2.3 GB episode store) exceed L2"},
        "ms_rollout": sum(roll_ms) / max(1, len(roll_ms)), "ms_update": ms_per_step - sum(roll_ms) / max(1, len(roll_ms)),
        "rollout_kernels_ms": breakdown, "update_phases_ms": upd, "aux_learners_ms": aux, "gpu_launches": launches, "clocks": clocks, "roofline": roofline, "e2e": e2e,
    }
    log("gpu legs done" + ("; cpu baseline" if world == 1 and not args.no_cpu_baseline else ""))
    if world == 1 and not args.no_cpu_baseline:
        from oracle import ref_driver as R
        if R.available():
            cpu, kind = R.measure(B=Bl, T=T), "reference"
        else:
            from oracle import cpu_baseline as cb
            from iplan_b200.config import make_args
            cpu, kind = cb.measure(make_args("highway", use_cuda=False, device="cpu"), B=Bl, rollout_steps=2, train_eps=32), "port"
        out["cpu_baseline"] = {"value": cpu["value"], "unit": "env-steps/s", "cores": cpu["cores"], "kind": kind,
                               "sample": cpu["sample"], "t_rollout_step_s": cpu["t_step"], "t_update_s": cpu["t_train"]}
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
