"""Batch-sharded RNN-T loss across GPUs (SURVEY.md §8(e)).

The reference is single-device; utterances are independent (reference cpu_rnnt.h:290-301 already
treats them so), so the multi-GPU path is a contiguous batch split with ONE all-reduce of
(sum of costs, number of utterances) per step over NCCL/NVLink.  Gradients stay in place on each
shard; for 'mean' they are scaled by 1/N_global (not 1/N_local) inside the gradient kernel.
"""
import torch
import torch.distributed as dist

from . import _RNNT, certify_inputs  # noqa: F401
from .warp_rnnt import grad_options, lattice_options, rnnt_type_code


def shard_bounds(n_global, rank, world):
    """Contiguous split of n_global utterances over `world` ranks; first (n % world) ranks get one more."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    base, rem = divmod(n_global, world)
    start = rank * base + min(rank, rem)
    return start, base + (1 if rank < rem else 0)


def reduce_loss(local_cost_sum, local_n, reduction='mean', group=None):
    """All-reduce (sum) of the pair (cost sum, utterance count); returns (global loss, N_global).

    local_cost_sum: 0-d or 1-element tensor on the compute device (CUDA with NCCL; CPU with gloo
    in the host-logic tests).  One collective of two floats per step."""
    if reduction not in ('sum', 'mean'):
        raise ValueError("reduction must be 'sum' or 'mean' for the sharded loss")
    pair = torch.stack((local_cost_sum.reshape(()).to(torch.float64),
                        torch.tensor(float(local_n), dtype=torch.float64, device=local_cost_sum.device)))
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(pair, op=dist.ReduceOp.SUM, group=group)
    total, n_global = pair[0], pair[1]
    loss = total / n_global if reduction == 'mean' else total
    return loss.to(local_cost_sum.dtype), int(round(float(n_global)))


class ShardedRNNTLoss(torch.nn.Module):
    """RNNTLoss over a batch that is split across the ranks of a process group.

    forward(acts, labels, act_lens, label_lens) takes THIS rank's shard and returns the global
    'sum' or 'mean' loss (identical on every rank).  backward leaves d(global loss)/d(acts) on the
    local shard.  n_global must be known up front for 'mean' (it fixes the gradient scale before
    the collective completes, so no host synchronisation is needed); pass None to infer it as
    world_size * local batch.  fastemit_lambda / clamp: the keyword-only gradient options of rnnt_loss; the
    clip applies to each utterance's gradient before the 1/N_global of 'mean'.  delay_penalty and rnnt_type:
    rnnt_loss's."""

    def __init__(self, blank=0, reduction='mean', group=None, n_global=None, *, fastemit_lambda=0.0, clamp=-1.0,
                 delay_penalty=0.0, rnnt_type='regular'):
        super().__init__()
        grad_options(fastemit_lambda, clamp)
        lattice_options(delay_penalty)
        rnnt_type_code(rnnt_type)
        self.rnnt_type = rnnt_type
        self.blank, self.reduction, self.group, self.n_global = blank, reduction, group, n_global
        self.fastemit_lambda, self.clamp = fastemit_lambda, clamp
        self.delay_penalty = delay_penalty

    def forward(self, acts, labels, act_lens, label_lens):
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        n_local = acts.size(0)
        n_global = self.n_global if self.n_global is not None else n_local * world
        local = _RNNT.apply(acts, labels, act_lens, label_lens, self.blank, 'sum', self.fastemit_lambda,
                            self.clamp, self.delay_penalty, self.rnnt_type)   # [1], grads unscaled
        if self.reduction == 'mean':
            local = local / n_global            # autograd carries the 1/N_global into backward
        if world > 1:
            total = local.detach().clone()
            dist.all_reduce(total, group=self.group)
            # value = global, gradient = local (each rank owns its shard's gradient)
            return local + (total - local.detach())
        return local
