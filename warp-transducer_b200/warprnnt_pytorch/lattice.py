"""The RNN-T loss, its gradient and forced alignment on caller-supplied log-probabilities (DESIGN.md §13; k2's
mutual_information_recursion).  For joiners and lattices the logits entries do not form: a HAT or blank-factorised
joiner, internal-LM subtraction or label priors, LM fusion before alignment, factors scattered from a pruned grid.

    loss = rnnt_lattice_loss(px, py, act_lens, label_lens)              # px [N, S, T], py [N, S+1, T]
    frames, scores = rnnt_lattice_forced_align(px, py, act_lens, label_lens)

px[b, s, t] is the log-probability of emitting label s at frame t from context s, py[b, s, t] the blank
log-probability at (t, s): k2's orientation, with k2's px[..., :T] (its column T is -inf in every k2 transducer loss).
Factors need not be normalised.  k2's constrained transducer is
rnnt_lattice_loss(px + py[:, 1:, :], py, act_lens, label_lens, rnnt_type='modified').
"""
import torch
from torch.autograd import Function
from torch.nn import Module

from . import warp_rnnt
from ._checks import LengthCheck, check_contiguous, check_dim, check_type

_FLOATS = (torch.float32, torch.float64, torch.bfloat16, torch.float16)


def _check_lattice_inputs(px, py, act_lens, label_lens, rnnt_type, reduction='none'):
    """rnnt_loss's rules and exception types, for factors: ValueError for a bad rnnt_type or reduction, TypeError for
    a dtype, ValueError for a rank, a shape or a non-contiguous length tensor, RuntimeError for a CPU tensor or a
    second device.  Returns the deferred T == max(act_lens), S == max(label_lens) check and contiguous px, py."""
    warp_rnnt.rnnt_type_code(rnnt_type)
    if reduction not in ('none', 'sum', 'mean'):
        raise ValueError("reduction must be 'none', 'sum' or 'mean'")
    if py.dtype not in _FLOATS:
        raise TypeError("unsupported data type %s" % py.dtype)
    if px.dtype is not py.dtype:
        raise TypeError("px and py must have the same dtype, got %s and %s" % (px.dtype, py.dtype))
    check_type(act_lens, torch.int32, "lengths")
    check_type(label_lens, torch.int32, "label_lengths")
    check_contiguous(act_lens, "lengths")
    check_contiguous(label_lens, "label_lengths")
    check_dim(px, 3, "px")
    check_dim(py, 3, "py")
    check_dim(act_lens, 1, "lengths")
    check_dim(label_lens, 1, "label_lengths")
    N, S, T = px.shape
    if tuple(py.shape) != (N, S + 1, T):
        raise ValueError("py must be [N, S+1, T] = %s for px [N, S, T] = %s, got %s"
                         % ([N, S + 1, T], list(px.shape), list(py.shape)))
    if T < 1:
        raise ValueError("px and py must have at least one frame")
    if act_lens.shape[0] != N:
        raise ValueError("must have a length per example.")
    if label_lens.shape[0] != N:
        raise ValueError("must have a label length per example.")
    if not (px.is_cuda and py.is_cuda):
        raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only; there is no CPU fallback")
    warp_rnnt.require_same_device(py, px=px, act_lens=act_lens, label_lens=label_lens)
    return LengthCheck(act_lens, label_lens, T, S + 1), px.contiguous(), py.contiguous()


class _RNNTLattice(Function):
    """forward: import the factors and run the wavefronts (2 launches), the workspace kept in ctx.  backward: one
    kernel writes both gradients from the workspace alone, grad_output and the 'mean' factor applied."""

    @staticmethod
    def forward(ctx, px, py, act_lens, label_lens, reduction, rnnt_type):
        length_check, pxc, pyc = _check_lattice_inputs(px, py, act_lens, label_lens, rnnt_type, reduction)
        N = py.size(0)
        need_grad = px.requires_grad or py.requires_grad
        costs = torch.empty(N, dtype=warp_rnnt.costs_dtype(py), device=py.device)
        ws = warp_rnnt.gpu_lattice_forward(pxc.detach(), pyc.detach(), act_lens, label_lens, costs,
                                           prepare_backward=need_grad, rnnt_type=rnnt_type)
        length_check.finish()
        if need_grad:
            ctx.save_for_backward(act_lens, label_lens)
            ctx.workspace = ws
            ctx.rnnt_type = rnnt_type
            ctx.shapes = (px.shape, py.shape, py.dtype)
            ctx.scale = 1.0 / N if reduction == 'mean' else 1.0
        if reduction in ('sum', 'mean'):
            costs = costs.sum().unsqueeze_(-1)
            if reduction == 'mean':
                costs /= N
        return costs

    @staticmethod
    def backward(ctx, grad_output):
        act_lens, label_lens = ctx.saved_tensors
        px_shape, py_shape, dtype = ctx.shapes
        n = py_shape[0]
        g = grad_output.reshape(-1).to(device=act_lens.device, dtype=torch.float64 if dtype == torch.float64
                                       else torch.float32)
        g = g.expand(n).contiguous() if g.numel() == 1 else g.contiguous()
        px_grad = torch.empty(px_shape, dtype=dtype, device=act_lens.device)   # every element is written
        py_grad = torch.empty(py_shape, dtype=dtype, device=act_lens.device)
        warp_rnnt.gpu_lattice_backward(px_grad, py_grad, act_lens, label_lens, g, ctx.scale, ctx.workspace,
                                       rnnt_type=ctx.rnnt_type)
        return (px_grad if ctx.needs_input_grad[0] else None, py_grad if ctx.needs_input_grad[1] else None,
                None, None, None, None)


def rnnt_lattice_loss(px, py, act_lens, label_lens, reduction='mean', *, rnnt_type='regular'):
    """RNN-T loss on caller-supplied natural-log factors: px [N, S, T] label, py [N, S+1, T] blank, one floating
    dtype (fp32, fp64, bf16, fp16; the 16-bit types compute in fp32), on one CUDA device; act_lens / label_lens
    int32 [N] with T == max(act_lens) and S == max(label_lens).  Non-contiguous factors are copied.

    Returns -log-likelihood per utterance ('none'; float32, float64 for fp64 factors), their sum or their mean.  An
    utterance without a path costs +inf and gets a zero gradient; a NaN or +inf factor makes its cost NaN.  The
    gradients are exact: d cost / d py = -(blank occupancy), d cost / d px = -(label occupancy), zero on padding.
    rnnt_type: 'regular' (k2's -mutual_information_recursion) or 'modified' (one symbol per frame)."""
    return _RNNTLattice.apply(px, py, act_lens, label_lens, reduction, rnnt_type)


class RNNTLatticeLoss(Module):
    """Module form of rnnt_lattice_loss: RNNTLatticeLoss(reduction='mean', *, rnnt_type='regular')."""

    def __init__(self, reduction='mean', *, rnnt_type='regular'):
        super().__init__()
        warp_rnnt.rnnt_type_code(rnnt_type)
        if reduction not in ('none', 'sum', 'mean'):
            raise ValueError("reduction must be 'none', 'sum' or 'mean'")
        self.reduction = reduction
        self.rnnt_type = rnnt_type

    def forward(self, px, py, act_lens, label_lens):
        return rnnt_lattice_loss(px, py, act_lens, label_lens, self.reduction, rnnt_type=self.rnnt_type)


def rnnt_lattice_forced_align(px, py, act_lens, label_lens, *, rnnt_type='regular'):
    """(frames, scores) of the best alignment on caller-supplied factors, with rnnt_forced_align's contract: frames
    [N, S] int32 (-1 past label_lens[b]), scores [N] the path's log-score (float32, float64 for fp64 factors); -inf
    and -1 without a path, NaN and -1 with a NaN or +inf factor.  Inputs and checks as rnnt_lattice_loss.  No
    autograd graph."""
    length_check, pxc, pyc = _check_lattice_inputs(px, py, act_lens, label_lens, rnnt_type)
    N, S, _ = px.shape
    frames = torch.empty((N, S), dtype=torch.int32, device=py.device)
    scores = torch.empty(N, dtype=warp_rnnt.costs_dtype(py), device=py.device)
    warp_rnnt.gpu_lattice_align(pxc.detach(), pyc.detach(), act_lens, label_lens, frames, scores,
                                rnnt_type=rnnt_type)
    length_check.finish()
    return frames, scores
