"""Host-side logic of the env-sharded (data-parallel) learner — new capability, the
reference has no distributed path (SURVEY §8e).

One process per GPU; rank r owns envs [r*B, (r+1)*B) for the rollout and keeps their
episodes for learning.  What must be global for N ranks x B envs to reproduce one rank x N*B
envs (reference lines in learners/ippo_learner.py):
  * the "first batch_size of buffer_size episodes are trained on" rule (:371-394)
  * advantage mean and UNBIASED std over all Bf*T entries (:278) and the mask sums that
    normalise the policy / value losses (:155, :193)          -> all-reduce of 4 doubles / agent
  * the gradients (then the clip norm, :205/:219, follows)      -> one all-reduce per PPO epoch
"""
import torch


def dist_or_none():
    import torch.distributed as dist
    return dist if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 else None


def shard_train_episodes(rank, world, eps_local, batch_size_global):
    """How many of this rank's `eps_local` episodes (taken from the front) are trained on,
    when globally the first `batch_size_global` of world*eps_local episodes are (rank-major
    order).  With the reference's batch_size = buffer_size - 1 only the last rank drops one."""
    return int(max(0, min(eps_local, batch_size_global - rank * eps_local)))


def local_minibatch_rows(perm, num_mini_batch, T, ep_lo, ep_hi):
    """A rank's share of the shuffled mini-batches (num_mini_batch > 1; generate_data, learners/ippo_learner.py:368-424).

    ``perm`` [..., n] holds global permutations of the training rows r = b * T + t (b a global episode, rank-major).
    Set m of a permutation is perm[m * mbs : (m + 1) * mbs], mbs = n // num_mini_batch; the n % num_mini_batch
    trailing entries belong to no set.  The rank that holds the training episodes [ep_lo, ep_hi) keeps, per set and in
    the permutation's order, the rows of its own episodes, renumbered (b - ep_lo) * T + t.

    Returns ``idx`` [..., num_mini_batch, cap] (cap = the rank's largest share of a set; shorter shares are padded with
    -1) and ``count`` [..., num_mini_batch].  Over the ranks the shares of a set add up to the set, whatever the sizes."""
    n = perm.shape[-1]
    mbs = n // num_mini_batch
    sets = perm[..., :num_mini_batch * mbs].reshape(*perm.shape[:-1], num_mini_batch, mbs).long()
    ep = sets // T
    mine = (ep >= ep_lo) & (ep < ep_hi)
    count = mine.sum(-1)
    cap = int(count.max()) if count.numel() else 0
    if cap == mbs and bool(mine.all()):
        return sets - ep_lo * T, count
    order = torch.argsort((~mine).to(torch.uint8), dim=-1, stable=True)[..., :cap]      # own rows first, order kept
    idx = torch.gather(sets - ep_lo * T, -1, order)
    pad = torch.arange(cap, device=perm.device) >= count.unsqueeze(-1)
    return idx.masked_fill(pad, -1), count


def allreduce_sum_(t):
    """In-place SUM all-reduce when a process group with >1 rank is active; no-op otherwise."""
    d = dist_or_none()
    if d is not None:
        d.all_reduce(t)
    return t


def advantage_norm_from_moments(moments, n_train_rows_global):
    """(mean, 1/(std+1e-5), 1/sum_alive, 1/n_rows) from summed moments [A,4] =
    (sum adv, sum adv^2, count, sum alive over training rows) — the arithmetic of
    csrc/learner.cu:adv_finalize_kernel, kept here for the CPU test of the sharded path."""
    m = moments.double()
    s1, s2, n, sm = m[:, 0], m[:, 1], m[:, 2], m[:, 3]
    mean = s1 / n
    var = ((s2 - n * mean * mean) / (n - 1.0)).clamp_min(0.0)
    return torch.stack([mean.float(), 1.0 / (var.sqrt().float() + 1e-5), (1.0 / sm).float(),
                        torch.full_like(mean, 1.0 / n_train_rows_global).float()], dim=1)


class GradBucket:
    """Actor + critic gradients of all agents as ONE flat buffer -> ONE collective per epoch."""

    def __init__(self):
        self.buf = None

    def allreduce(self, grads):
        d = dist_or_none()
        if d is None:
            return
        n = sum(g.numel() for g in grads)
        if self.buf is None or self.buf.numel() != n or self.buf.device != grads[0].device:
            self.buf = torch.empty(n, dtype=grads[0].dtype, device=grads[0].device)
        o = 0
        for g in grads:
            self.buf[o:o + g.numel()].copy_(g.reshape(-1))
            o += g.numel()
        d.all_reduce(self.buf)
        o = 0
        for g in grads:
            g.view(-1).copy_(self.buf[o:o + g.numel()])
            o += g.numel()
