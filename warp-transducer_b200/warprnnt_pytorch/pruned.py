"""Pruned RNN-T loss (Kuang et al., "Pruned RNN-T for fast, memory-efficient ASR training", Interspeech 2022),
with the pruning ranges taken from the additive joint's lattice (DESIGN.md §8).

A training step with a real (nonlinear) joiner:

    simple, ranges = add_joint_rnnt_loss_with_ranges(am_proj, lm_proj, labels, act_lens, label_lens, s_range=5)
    enc_p, dec_p = prune_joint_inputs(enc, dec, ranges, s_range=5)          # [N,T,R,D] each
    logits = joiner(enc_p, dec_p)                                             # [N,T,R,V]
    pruned = pruned_rnnt_loss(logits, labels, act_lens, label_lens, ranges)
    (simple_scale * simple + pruned).backward()

The pruned loss reads R logits per frame instead of U: row (b, t, s) of `logits` is lattice cell
(t, ranges[b, t] + s).  Cells no row covers cannot be visited; rows outside the utterance get a zero gradient.

For icefall's joiner, logits = W act(enc + pred) + bias, the middle three lines are one call that never forms the
[N, T, R, V] logits: pruned_joiner_rnnt_loss(enc, pred, W, bias, labels, act_lens, label_lens, ranges, 5)
(joiner.py, DESIGN.md §15).
"""
import ctypes as C

import torch
from torch.autograd import Function
from torch.nn import Module

from . import warp_rnnt
from ._checks import LengthCheck, check_contiguous, check_dim, check_type
from .joint import _AddJointRNNT, _joint_opts, _lab_ptr, check_joint_call, joint_forward_call

_lib = warp_rnnt.lib()
_P = C.c_void_p
_Opt, _GOpt = warp_rnnt.rnntOptions, warp_rnnt.rnntGradOptions
_lib.rnnt_b200_pruned_workspace_size.restype = C.c_int
_lib.rnnt_b200_pruned_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t,
                                                 C.POINTER(C.c_size_t)]
_lib.rnnt_b200_pruned_loss_async_ex.restype = C.c_int
_lib.rnnt_b200_pruned_loss_async_ex.argtypes = [C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int,
                                                _P, C.c_double, _GOpt, _P, _Opt]
_lib.rnnt_b200_pruned_forward.restype = C.c_int
_lib.rnnt_b200_pruned_forward.argtypes = [C.c_int, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P,
                                          _Opt]
_lib.rnnt_b200_pruned_backward_ex.restype = C.c_int
_lib.rnnt_b200_pruned_backward_ex.argtypes = [C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P,
                                              C.c_double, _GOpt, _P, _Opt]
_LOpt = warp_rnnt.rnntLatticeOptions
_lib.rnnt_b200_pruned_forward_lat.restype = C.c_int
_lib.rnnt_b200_pruned_forward_lat.argtypes = [C.c_int, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int,
                                              _LOpt, _P, _Opt]
_lib.rnnt_b200_pruned_backward_lat.restype = C.c_int
_lib.rnnt_b200_pruned_backward_lat.argtypes = [C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P,
                                               C.c_double, _GOpt, _LOpt, _P, _Opt]
_lib.rnnt_b200_pruned_loss_async_lat.restype = C.c_int
_lib.rnnt_b200_pruned_loss_async_lat.argtypes = [C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int,
                                                 C.c_int, _P, C.c_double, _GOpt, _LOpt, _P, _Opt]
_lib.rnnt_b200_pruned_forward_topo.restype = C.c_int
_lib.rnnt_b200_pruned_forward_topo.argtypes = [C.c_int, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int,
                                               _LOpt, C.c_int, _P, _Opt]
_lib.rnnt_b200_pruned_backward_topo.restype = C.c_int
_lib.rnnt_b200_pruned_backward_topo.argtypes = [C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P,
                                                C.c_double, _GOpt, _LOpt, C.c_int, _P, _Opt]
_lib.rnnt_b200_pruned_loss_async_topo.restype = C.c_int
_lib.rnnt_b200_pruned_loss_async_topo.argtypes = [C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int,
                                                  C.c_int, _P, C.c_double, _GOpt, _LOpt, C.c_int, _P, _Opt]
_lib.rnnt_b200_add_joint_prune_ranges.restype = C.c_int
_lib.rnnt_b200_add_joint_prune_ranges.argtypes = [_P, _P, C.c_int, C.c_int, _P, _P, _Opt]
_lib.rnnt_b200_add_joint_prune_ranges_topo.restype = C.c_int
_lib.rnnt_b200_add_joint_prune_ranges_topo.argtypes = [_P, _P, C.c_int, C.c_int, _P, _P, C.c_int, _Opt]
_lib.rnnt_b200_add_joint_workspace_size.restype = C.c_int


def pruned_workspace_size(maxT, maxU, s_range, minibatch, dtype_size=4):
    n = C.c_size_t(0)
    st = _lib.rnnt_b200_pruned_workspace_size(maxT, maxU, s_range, minibatch, dtype_size, C.byref(n))
    if st != 0:
        raise ValueError("rnnt_b200_pruned_workspace_size: " + warp_rnnt.status_string(st))
    return n.value


# ---- pruning ranges from the additive joint -------------------------------------------------------------------
class _AddJointRNNTRanges(Function):
    """_AddJointRNNT's forward with beta always kept, plus the ranges kernel on its workspace; the same backward."""

    @staticmethod
    def forward(ctx, trans, pred, labels, act_lens, label_lens, blank, reduction, fastemit_lambda, s_range,
                lm_only_scale=0.0, am_only_scale=0.0, delay_penalty=0.0, rnnt_type='regular'):
        s_range = int(s_range)
        if s_range < 2:
            raise ValueError("s_range must be >= 2, got %d" % s_range)
        lattice = warp_rnnt.lattice_options(delay_penalty)
        topo = warp_rnnt.rnnt_type_code(rnnt_type)
        gopt, smooth, length_check = check_joint_call(trans, pred, labels, act_lens, label_lens, reduction,
                                                      fastemit_lambda, lm_only_scale, am_only_scale)
        N, T = trans.shape[0], trans.shape[1]
        length_check.guard_labels(labels, N)
        costs = torch.empty(N, dtype=torch.float32, device=trans.device)
        ranges = torch.empty((N, T), dtype=torch.int32, device=trans.device)
        with torch.cuda.device(trans.device):
            ws = joint_forward_call(trans, pred, labels, act_lens, label_lens, costs, True, blank, smooth, lattice,
                                    topo)
            if topo != warp_rnnt.RNNT_B200_RNNT_REGULAR:
                st = _lib.rnnt_b200_add_joint_prune_ranges_topo(label_lens.data_ptr(), act_lens.data_ptr(), N,
                                                                s_range, ranges.data_ptr(), ws.data_ptr(), topo,
                                                                _joint_opts(trans, pred, blank))
            else:
                st = _lib.rnnt_b200_add_joint_prune_ranges(label_lens.data_ptr(), act_lens.data_ptr(), N, s_range,
                                                           ranges.data_ptr(), ws.data_ptr(),
                                                           _joint_opts(trans, pred, blank))
        if st != 0:
            raise RuntimeError("rnnt_b200_add_joint_prune_ranges failed: " + warp_rnnt.status_string(st))
        length_check.finish()
        ctx.mark_non_differentiable(ranges)
        ctx.save_for_backward(trans, pred, labels, act_lens, label_lens)
        ctx.ws, ctx.blank, ctx.gopt, ctx.smooth, ctx.topo = ws, blank, gopt, smooth, topo
        ctx.scale = 1.0 / N if reduction == 'mean' else 1.0
        if reduction in ('sum', 'mean'):
            costs = costs.sum().unsqueeze_(-1)
            if reduction == 'mean':
                costs /= N
        return costs, ranges

    @staticmethod
    def backward(ctx, grad_output, grad_ranges):
        dtrans, dpred = _AddJointRNNT.backward(ctx, grad_output)[:2]
        return dtrans, dpred, None, None, None, None, None, None, None, None, None, None, None


def add_joint_rnnt_loss_with_ranges(trans, pred, labels, act_lens, label_lens, s_range, blank=0, reduction='mean',
                                    *, fastemit_lambda=0.0, lm_only_scale=0.0, am_only_scale=0.0, delay_penalty=0.0,
                                    rnnt_type='regular'):
    """(loss, ranges): add_joint_rnnt_loss (the "simple" loss of pruned RNN-T; differentiable in trans and pred
    exactly as add_joint_rnnt_loss) and the [N, T] int32 window starts of the pruned loss for R = s_range >= 2,
    from the same forward (include/rnnt.h, rnnt_b200_add_joint_prune_ranges, defines them).  lm_only_scale and
    am_only_scale smooth the simple loss as add_joint_rnnt_loss's do (icefall's --lm-scale / --am-scale); the
    windows then come from the smoothed lattice.  delay_penalty penalises it as add_joint_rnnt_loss's does (icefall's
    --delay-penalty), and the windows come from the penalised lattice, as k2's do.  rnnt_type: rnnt_loss's; the
    windows of a 'modified' lattice come from its own occupancies and may leave an utterance no path through the
    pruned modified loss (DESIGN.md §11)."""
    return _AddJointRNNTRanges.apply(trans, pred, labels, act_lens, label_lens, blank, reduction, fastemit_lambda,
                                     s_range, lm_only_scale, am_only_scale, delay_penalty, rnnt_type)


def prune_joint_inputs(enc, dec, ranges, s_range):
    """The joiner's inputs at the pruned cells: enc [N,T,D] expanded (no copy) and dec [N,U,D] gathered at
    clamp(ranges + s, 0, U-1), both [N, T, s_range, D].  Rows whose u is clamped are padding to the pruned loss, so
    what they hold does not matter.  (k2's do_rnnt_pruning, torch only.)"""
    N, T, D = enc.shape
    U = dec.shape[1]
    R = int(s_range)
    if ranges.shape != (N, T):
        raise ValueError("ranges must be [N, T] = [%d, %d], got %s" % (N, T, tuple(ranges.shape)))
    idx = (ranges.long().unsqueeze(-1) + torch.arange(R, device=ranges.device)).clamp_(0, U - 1)   # [N,T,R]
    dec_p = torch.gather(dec.unsqueeze(1).expand(N, T, U, D), 2, idx.unsqueeze(-1).expand(N, T, R, D))
    return enc.unsqueeze(2).expand(N, T, R, D), dec_p


# ---- pruned loss ------------------------------------------------------------------------------------------------
def _check_pruned_inputs(logits, labels, act_lens, label_lens, ranges):
    """RNNTLoss's input rules for [N, T, R, V] logits (U comes from labels), plus the ranges."""
    named = (("logits", logits, None, 4), ("labels", labels, torch.int32, 2),
             ("lengths", act_lens, torch.int32, 1), ("label_lengths", label_lens, torch.int32, 1),
             ("ranges", ranges, torch.int32, 2))
    for name, tensor, dtype, _ in named:
        if dtype is not None:
            check_type(tensor, dtype, name)
    for name, tensor, _, _ in named:
        check_contiguous(tensor, name)
    for name, tensor, _, rank in named:
        check_dim(tensor, rank, name)
    N, T = logits.shape[0], logits.shape[1]
    if act_lens.shape[0] != N:
        raise ValueError("must have a length per example.")
    if label_lens.shape[0] != N:
        raise ValueError("must have a label length per example.")
    if tuple(ranges.shape) != (N, T):
        raise ValueError("ranges must be [N, T] = [%d, %d], got %s" % (N, T, tuple(ranges.shape)))
    if not logits.is_cuda:
        raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only; there is no CPU fallback")
    warp_rnnt.require_same_device(logits, labels=labels, act_lens=act_lens, label_lens=label_lens, ranges=ranges)
    return LengthCheck(act_lens, label_lens, T, labels.shape[1] + 1)


def _opts(logits, blank, maxU):
    return _Opt(loc=1, num_threads=0, stream=torch.cuda.current_stream(logits.device).cuda_stream,
                blank_label=blank, maxT=logits.shape[1], maxU=maxU, batch_first=True)


class _PrunedRNNT(Function):
    """_RNNT's split for [N, T, R, V] logits: forward = statistics of the rows + the pruned lattices, backward =
    the gradient pass with grad_output and the 'mean' factor folded in."""

    @staticmethod
    def forward(ctx, logits, labels, act_lens, label_lens, ranges, blank, reduction, fastemit_lambda=0.0,
                clamp=-1.0, delay_penalty=0.0, rnnt_type='regular'):
        warp_rnnt.grad_options(fastemit_lambda, clamp)   # ValueError before any device work
        lattice = warp_rnnt.lattice_options(delay_penalty)
        topo = warp_rnnt.rnnt_type_code(rnnt_type)
        code = warp_rnnt._dtype_code(logits)
        if reduction not in ('none', 'sum', 'mean'):
            raise ValueError("reduction must be 'none', 'sum' or 'mean'")
        length_check = _check_pruned_inputs(logits, labels, act_lens, label_lens, ranges)
        N, T, R, V = logits.shape
        U = labels.shape[1] + 1
        length_check.guard_labels(labels, N)
        need_grad = logits.requires_grad
        costs = torch.empty(N, dtype=warp_rnnt.costs_dtype(logits), device=logits.device)
        with torch.cuda.device(logits.device):
            ws = torch.empty(pruned_workspace_size(T, U, R, N, 8 if logits.dtype == torch.float64 else 4),
                             dtype=torch.uint8, device=logits.device)
            args = (code, logits.data_ptr(), ranges.data_ptr(), R, _lab_ptr(labels), label_lens.data_ptr(),
                    act_lens.data_ptr(), V, N, costs.data_ptr(), 1 if need_grad else 0)
            tail = (ws.data_ptr(), _opts(logits, blank, U))
            if topo != warp_rnnt.RNNT_B200_RNNT_REGULAR:
                st = _lib.rnnt_b200_pruned_forward_topo(*args, lattice or _LOpt(), topo, *tail)
            elif lattice is None:
                st = _lib.rnnt_b200_pruned_forward(*args, *tail)
            else:
                st = _lib.rnnt_b200_pruned_forward_lat(*args, lattice, *tail)
        if st != 0:
            raise RuntimeError("rnnt_b200_pruned_forward failed: " + warp_rnnt.status_string(st))
        length_check.finish()
        if need_grad:
            ctx.save_for_backward(logits, labels, act_lens, label_lens, ranges)
            ctx.workspace, ctx.blank, ctx.maxU = ws, blank, U
            ctx.fastemit_lambda, ctx.clamp, ctx.lattice, ctx.topo = fastemit_lambda, clamp, lattice, topo
            ctx.scale = 1.0 / N if reduction == 'mean' else 1.0
        if reduction in ('sum', 'mean'):
            costs = costs.sum().unsqueeze_(-1)
            if reduction == 'mean':
                costs /= N
        return costs

    @staticmethod
    def backward(ctx, grad_output):
        logits, labels, act_lens, label_lens, ranges = ctx.saved_tensors
        N, T, R, V = logits.shape
        g = grad_output.reshape(-1).to(device=logits.device, dtype=warp_rnnt.costs_dtype(logits))
        g = g.expand(N).contiguous() if g.numel() == 1 else g.contiguous()
        grads = torch.empty_like(logits)   # the kernel defines every element (zeros on padding)
        gopt = warp_rnnt._ex_options(ctx.fastemit_lambda, ctx.clamp)
        with torch.cuda.device(logits.device):
            args = (warp_rnnt._dtype_code(logits), logits.data_ptr(), grads.data_ptr(), ranges.data_ptr(), R,
                    _lab_ptr(labels), label_lens.data_ptr(), act_lens.data_ptr(), V, N, g.data_ptr(), ctx.scale, gopt)
            tail = (ctx.workspace.data_ptr(), _opts(logits, ctx.blank, ctx.maxU))
            if ctx.topo != warp_rnnt.RNNT_B200_RNNT_REGULAR:
                st = _lib.rnnt_b200_pruned_backward_topo(*args, ctx.lattice or _LOpt(), ctx.topo, *tail)
            elif ctx.lattice is None:
                st = _lib.rnnt_b200_pruned_backward_ex(*args, *tail)
            else:
                st = _lib.rnnt_b200_pruned_backward_lat(*args, ctx.lattice, *tail)
        if st != 0:
            raise RuntimeError("rnnt_b200_pruned_backward_ex failed: " + warp_rnnt.status_string(st))
        return grads, None, None, None, None, None, None, None, None, None, None


def pruned_rnnt_loss(logits, labels, act_lens, label_lens, ranges, blank=0, reduction='mean', *,
                     fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0, rnnt_type='regular'):
    """Pruned RNN-T loss of logits [N, T, R, V] (fp32 / fp64 / bf16 / fp16), row (b, t, s) = lattice cell
    (t, ranges[b, t] + s); ranges [N, T] int32 on the logits' device.  labels, lengths, reduction and the gradient
    options are rnnt_loss's; the lattice is [T, max(label_lens) + 1] as there.  An utterance whose windows leave no
    path costs +inf with a zero gradient.  With R = U and ranges == 0 this is rnnt_loss exactly.  delay_penalty:
    rnnt_loss's, on the covered cells (icefall passes the same value to the simple and the pruned loss).
    rnnt_type: rnnt_loss's; with 'modified' the windows may leave an utterance no path (DESIGN.md §11)."""
    return _PrunedRNNT.apply(logits, labels, act_lens, label_lens, ranges, blank, reduction, fastemit_lambda, clamp,
                             delay_penalty, rnnt_type)


class PrunedRNNTLoss(Module):
    """Module form of pruned_rnnt_loss: PrunedRNNTLoss(blank=0, reduction='mean', *, fastemit_lambda=0.0,
    clamp=-1.0, delay_penalty=0.0, rnnt_type='regular')(logits, labels, act_lens, label_lens, ranges)."""

    def __init__(self, blank=0, reduction='mean', *, fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0,
                 rnnt_type='regular'):
        super().__init__()
        warp_rnnt.grad_options(fastemit_lambda, clamp)
        warp_rnnt.lattice_options(delay_penalty)
        warp_rnnt.rnnt_type_code(rnnt_type)
        self.blank, self.reduction = blank, reduction
        self.fastemit_lambda, self.clamp, self.delay_penalty = fastemit_lambda, clamp, delay_penalty
        self.rnnt_type = rnnt_type

    def forward(self, logits, labels, act_lens, label_lens, ranges):
        return _PrunedRNNT.apply(logits, labels, act_lens, label_lens, ranges, self.blank, self.reduction,
                                 self.fastemit_lambda, self.clamp, self.delay_penalty, self.rnnt_type)
