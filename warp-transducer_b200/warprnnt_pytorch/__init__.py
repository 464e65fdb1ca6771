"""warprnnt_pytorch — RNN-T loss operator for PyTorch on the H100-native libwarprnnt.

Same public surface as the reference package (pytorch_binding/warprnnt_pytorch/__init__.py):
``RNNTLoss(blank=0, reduction='mean')``, ``rnnt_loss(acts, labels, act_lens, label_lens,
blank=0, reduction='mean')`` and the ``warp_rnnt`` extension functions, with the reference's
input rules and error types (certify_inputs, :115-140).  Keyword-only additions:
``fastemit_lambda`` (FastEmit regularisation), ``clamp`` (element-wise gradient clipping),
``delay_penalty`` (the delay-penalised lattice of low-latency streaming training) and ``rnnt_type``
(k2's 'regular' or 'modified' one-symbol-per-frame topology); see rnnt_loss.  ``rnnt_forced_align`` and
``pruned_rnnt_forced_align`` give the best path's label frames and score (forced alignment).  ``rnnt_lattice_loss``,
``RNNTLatticeLoss`` and ``rnnt_lattice_forced_align`` run the loss, gradient and alignment on blank and label
log-probabilities the caller formed (k2's mutual_information_recursion).  Differences, all on the fast side:
the call never synchronises with the host except for the reference's own length check, costs
stay on the device, and the gradient is produced in autograd's backward with grad_output and the
'mean' factor folded into the kernel - no zeros_like / mul_ passes over the [N,T,U,V] tensor.
CPU tensors are rejected: there is no host path.
"""
import torch
from torch.autograd import Function
from torch.nn import Module

from . import warp_rnnt
from .warp_rnnt import cpu_rnnt, gpu_rnnt, gpu_rnnt_async, gpu_rnnt_backward, gpu_rnnt_forward  # noqa: F401

__all__ = ['rnnt_loss', 'RNNTLoss']


class _RNNT(Function):
    """One training step costs the algorithmic 12 B per logit: forward() reads the logits once
    (statistics + alpha/beta lattices, 4 B), backward() reads them again and writes the gradient
    with the upstream gradient and the 'mean' factor already applied (8 B).  The reference makes
    four more full-tensor passes around its C call (zeros_like, memset, grads /= N, grads.mul_)."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, blank, reduction, fastemit_lambda=0.0, clamp=-1.0,
                delay_penalty=0.0, rnnt_type='regular'):
        """
        acts: (batch x seqLength x labelLength x outputDim) raw joint-network logits
        labels: (batch x maxLabelLength) int32 targets, zero padded
        act_lens / label_lens: (batch) int32
        """
        warp_rnnt.grad_options(fastemit_lambda, clamp)   # ValueError before any device work
        warp_rnnt.lattice_options(delay_penalty)
        warp_rnnt.rnnt_type_code(rnnt_type)
        length_check = certify_inputs(acts, labels, act_lens, label_lens, defer=True)
        if not acts.is_cuda:
            raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only; "
                               "there is no CPU fallback")
        warp_rnnt.require_same_device(acts, labels=labels, act_lens=act_lens, label_lens=label_lens)
        if reduction not in ('none', 'sum', 'mean'):
            raise ValueError("reduction must be 'none', 'sum' or 'mean'")
        minibatch_size = acts.size(0)
        length_check.guard_labels(labels, minibatch_size)
        need_grad = acts.requires_grad
        # bf16 / fp16 logits: arithmetic, lattice and costs are fp32 (6 B per logit instead of 12)
        costs = torch.empty(minibatch_size, dtype=warp_rnnt.costs_dtype(acts), device=acts.device)
        ws = warp_rnnt.gpu_rnnt_forward(acts, labels, act_lens, label_lens, costs, blank,
                                        prepare_backward=need_grad, delay_penalty=delay_penalty, rnnt_type=rnnt_type)
        length_check.finish()   # T == max(act_lens), U == max(label_lens) + 1: waited for with the kernels queued
        if need_grad:
            ctx.save_for_backward(acts, labels, act_lens, label_lens)
            ctx.workspace = ws
            ctx.blank = blank
            ctx.fastemit_lambda, ctx.clamp, ctx.delay_penalty = fastemit_lambda, clamp, delay_penalty
            ctx.rnnt_type = rnnt_type
            # reference :38-40 divides costs and grads by N for 'mean'
            ctx.scale = 1.0 / minibatch_size if reduction == 'mean' else 1.0
        if reduction in ('sum', 'mean'):
            costs = costs.sum().unsqueeze_(-1)
            if reduction == 'mean':
                costs /= minibatch_size
        return costs

    @staticmethod
    def backward(ctx, grad_output):
        # reference :47-50: grads.mul_(grad_output.view(-1,1,1,1)); here the factor rides in the kernel
        acts, labels, act_lens, label_lens = ctx.saved_tensors
        n = acts.size(0)
        g = grad_output.reshape(-1).to(device=acts.device, dtype=warp_rnnt.costs_dtype(acts))
        g = g.expand(n).contiguous() if g.numel() == 1 else g.contiguous()
        grads = torch.empty_like(acts)   # the kernel defines every element (zeros on padding)
        warp_rnnt.gpu_rnnt_backward(acts, labels, act_lens, label_lens, grads, g, ctx.blank,
                                    ctx.scale, ctx.workspace, fastemit_lambda=ctx.fastemit_lambda,
                                    clamp=ctx.clamp, delay_penalty=ctx.delay_penalty, rnnt_type=ctx.rnnt_type)
        return grads, None, None, None, None, None, None, None, None, None


def rnnt_loss(acts, labels, act_lens, label_lens, blank=0, reduction='mean', *, fastemit_lambda=0.0,
              clamp=-1.0, delay_penalty=0.0, rnnt_type='regular'):
    """RNN Transducer loss (reference :53-70).

    reduction: 'none' | 'sum' | 'mean'; 'mean' divides the summed loss by the batch size (what
    the reference computes, :36-40).

    fastemit_lambda: FastEmit regularisation (Yu et al., ICASSP 2021), finite and >= 0; 0 = off.  The
    gradient with respect to each label log-probability is scaled by (1 + fastemit_lambda), which
    favours emitting labels early.  The returned loss is still the plain negative log-likelihood, so
    with fastemit_lambda > 0 the gradient is deliberately NOT the gradient of the returned loss
    (torch.autograd.gradcheck does not apply).
    clamp: > 0 clips every element of each utterance's logits gradient to [-clamp, clamp], before the
    upstream gradient and the 'mean' factor are applied (as torchaudio's rnnt_loss); <= 0 = off.
    delay_penalty: the delay-penalised transducer (Kang et al., ICASSP 2023; k2's delay_penalty), finite and
    >= 0; 0 = off.  Every label factor at frame t gains delay_penalty * ((T_b - 1)/2 - t), T_b the utterance's
    frame count; the returned loss includes the penalty (it can be negative) and the gradient is its exact
    gradient.  It favours emitting labels early (include/rnnt.h, rnntLatticeOptions).
    rnnt_type: 'regular' (default) or 'modified', k2's one-symbol-per-frame transducer: every frame takes exactly
    one transition, a blank or the next label, so a frame emits at most one label.  An utterance with more labels
    than frames then has no path: its loss is +inf and its gradient zero.  'constrained' is not supported.
    Invalid values raise ValueError.
    """
    return _RNNT.apply(acts, labels, act_lens, label_lens, blank, reduction, fastemit_lambda, clamp, delay_penalty,
                       rnnt_type)


class RNNTLoss(Module):
    """Module form (reference :73-100): RNNTLoss(blank=0, reduction='mean', *, fastemit_lambda=0.0,
    clamp=-1.0, delay_penalty=0.0, rnnt_type='regular'); the keyword-only options are those of rnnt_loss."""

    def __init__(self, blank=0, reduction='mean', *, fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0,
                 rnnt_type='regular'):
        super(RNNTLoss, self).__init__()
        warp_rnnt.grad_options(fastemit_lambda, clamp)
        warp_rnnt.lattice_options(delay_penalty)
        warp_rnnt.rnnt_type_code(rnnt_type)
        self.blank = blank
        self.reduction = reduction
        self.fastemit_lambda, self.clamp = fastemit_lambda, clamp
        self.delay_penalty = delay_penalty
        self.rnnt_type = rnnt_type
        self.loss = _RNNT.apply

    def forward(self, acts, labels, act_lens, label_lens):
        return self.loss(acts, labels, act_lens, label_lens, self.blank, self.reduction, self.fastemit_lambda,
                         self.clamp, self.delay_penalty, self.rnnt_type)


from ._checks import certify_inputs, check_contiguous, check_dim, check_type  # noqa: E402,F401
from .pruned import (PrunedRNNTLoss, add_joint_rnnt_loss_with_ranges, prune_joint_inputs,  # noqa: E402
                     pruned_rnnt_loss)

__all__ += ['pruned_rnnt_loss', 'PrunedRNNTLoss', 'add_joint_rnnt_loss_with_ranges', 'prune_joint_inputs']
from .align import pruned_rnnt_forced_align, rnnt_forced_align  # noqa: E402

__all__ += ['rnnt_forced_align', 'pruned_rnnt_forced_align']
from .lattice import RNNTLatticeLoss, rnnt_lattice_forced_align, rnnt_lattice_loss  # noqa: E402

__all__ += ['rnnt_lattice_loss', 'RNNTLatticeLoss', 'rnnt_lattice_forced_align']
from .joiner import (JoinerRNNTLoss, PrunedJoinerRNNTLoss, joiner_log_probs, joiner_rnnt_loss,  # noqa: E402
                     pruned_joiner_log_probs, pruned_joiner_rnnt_loss)

__all__ += ['joiner_log_probs', 'joiner_rnnt_loss', 'JoinerRNNTLoss', 'pruned_joiner_log_probs',
            'pruned_joiner_rnnt_loss', 'PrunedJoinerRNNTLoss']
