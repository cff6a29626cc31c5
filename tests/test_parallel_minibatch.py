"""Sharding of the shuffled mini-batches over ranks (iplan_b200.parallel.local_minibatch_rows) on the CPU: the ranks'
shares reassemble every set, a rank may hold nothing of a set, and two gloo ranks that run the float64 oracle on their
shares with the global denominators and all-reduce through GradBucket reproduce the unsharded mini-batch step."""
import os
import socket
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from iplan_b200 import parallel
from oracle import iplan_oracle as O
from oracle import minibatch_oracle as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "learner_minibatch.pt")


def _blocks(world, eps_local, batch_size):
    return [(r * eps_local, r * eps_local + parallel.shard_train_episodes(r, world, eps_local, batch_size)) for r in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_shares_reassemble_every_set(world):
    T, eps_local, k = 5, 4, 4
    batch_size = world * eps_local - 1
    n = batch_size * T
    g = torch.Generator().manual_seed(world)
    perm = torch.stack([torch.stack([torch.randperm(n, generator=g) for _ in range(3)]) for _ in range(2)])   # [A=2][E=3][n]
    mbs = n // k
    shares = [parallel.local_minibatch_rows(perm, k, T, lo, hi) for lo, hi in _blocks(world, eps_local, batch_size)]
    total = sum(c for _, c in shares)
    assert bool((total == mbs).all())
    for a in range(2):
        for e in range(3):
            for m in range(k):
                want = perm[a, e, m * mbs:(m + 1) * mbs]
                got = []
                for (idx, count), (lo, hi) in zip(shares, _blocks(world, eps_local, batch_size)):
                    c = int(count[a, e, m])
                    rows = idx[a, e, m, :c]
                    assert bool((idx[a, e, m, c:] == -1).all()) and bool((rows >= 0).all()) and bool((rows < (hi - lo) * T).all())
                    glob = rows + lo * T
                    # the share keeps the permutation's order
                    assert torch.equal(glob, want[(want // T >= lo) & (want // T < hi)])
                    got.append(glob)
                assert torch.equal(torch.cat(got).sort().values, want.sort().values)


def test_empty_local_set():
    T, k = 3, 2
    perm = torch.tensor([[0, 1, 2, 3, 4, 5, 6]])          # 2 sets of 3 rows (row 6 dropped): episodes 0 | 1
    idx, count = parallel.local_minibatch_rows(perm, k, T, 1, 2)
    assert count.tolist() == [[0, 3]]
    assert idx.tolist() == [[[-1, -1, -1], [0, 1, 2]]]
    idx, count = parallel.local_minibatch_rows(perm, k, T, 2, 3)      # holds only the dropped row
    assert count.tolist() == [[0, 0]] and idx.shape[-1] == 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _case():
    from tests.golden.minibatch_fixture import load
    g = load(GOLDEN)
    args = SimpleNamespace(**g["args"])
    ap = {k: v.double() for k, v in g["actors_before"][0].items()}
    cp = {k: v.double() for k, v in g["critics_before"][0].items()}
    flat = M.agent_rows(ap, cp, M.agent_batch(g["data"], 0, args.n_actions, torch.float64), 0, args)
    return args, ap, cp, flat, g["perms"][0, 0]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        args, ap, cp, flat, perm = _case()
        T, k = args.episode_limit, args.num_mini_batch
        eps_local = args.buffer_size // world
        lo = rank * eps_local
        hi = lo + parallel.shard_train_episodes(rank, world, eps_local, args.batch_size)
        idx, count = parallel.local_minibatch_rows(perm, k, T, lo, hi)
        res = []
        for m in range(k):
            rows = idx[m, :int(count[m])] + lo * T
            asum = flat["alive"][rows].sum().view(1)
            parallel.allreduce_sum_(asum)                                    # the set's global sum(alive)
            e = M.ppo_set(ap, cp, flat, args, rows, alive_sum=float(asum), n_rows=perm.shape[0] // k)
            ga = [e["grads_actor"][key].clone() for key in O.ACTOR_TRAINABLE]
            gc = [e["grads_critic"][key].clone() for key in O.CRITIC_TRAINABLE]
            parallel.GradBucket().allreduce(ga + gc)
            sc = torch.stack([e["policy_loss"], e["value_loss"], e["dist_entropy"], e["ratio"]]).double()
            parallel.allreduce_sum_(sc)
            res.append(([x.numpy() for x in ga], [x.numpy() for x in gc], sc.numpy()))      # numpy: pickled by value
        out.put((rank, [int(c) for c in count], res if rank == 0 else None))
    finally:
        dist.destroy_process_group()


def test_two_rank_mini_batch_step_equals_single_rank():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r, (c, x)) for r, c, x in (q.get(timeout=180) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    args, ap, cp, flat, perm = _case()
    k = args.num_mini_batch
    mbs = perm.shape[0] // k
    assert [a + b for a, b in zip(res[0][0], res[1][0])] == [mbs] * k
    for m, (ga, gc, sc) in enumerate(res[0][1]):
        e = M.ppo_set(ap, cp, flat, args, perm[m * mbs:(m + 1) * mbs])
        for kind, keys, grads in (("grads_actor", O.ACTOR_TRAINABLE, ga), ("grads_critic", O.CRITIC_TRAINABLE, gc)):
            for key, got in zip(keys, grads):
                ref, got = e[kind][key], torch.as_tensor(got)
                assert float((got - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), (m, kind, key)
        ref = torch.stack([e["policy_loss"], e["value_loss"], e["dist_entropy"], e["ratio"]]).double()
        assert float((torch.as_tensor(sc) - ref).abs().max()) < 1e-12, (m, sc, ref)
