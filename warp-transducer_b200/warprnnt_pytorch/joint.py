"""RNN-T loss for an ADDITIVE joint network without materialising the [N,T,U,V] logits
(SURVEY.md §8(f).2).  The reference's own timing script forms its logits as
``acts = trans.unsqueeze(2) + pred.unsqueeze(1)`` (pytorch_binding/test/test_time.py:73) and then
calls RNNTLoss on the 4-D tensor; this operator takes the two factors directly:

    loss = AddJointRNNTLoss(blank=0, reduction='mean')(trans, pred, labels, act_lens, label_lens)

trans [N,T,V], pred [N,U,V] fp32 CUDA, same label/length conventions and input checks as RNNTLoss.
Equivalent to RNNTLoss()(trans.unsqueeze(2) + pred.unsqueeze(1), ...) with gradients reduced to
the factors, at O(N (T+U) V) memory traffic.  The keyword-only ``fastemit_lambda`` is RNNTLoss's
FastEmit option; ``clamp`` is not available here (the factor gradients are contractions over the
lattice, per-logit gradients never exist to be clipped) and raises ValueError.

The keyword-only ``lm_only_scale`` and ``am_only_scale`` give k2's smoothed loss (rnnt_loss_smoothed, the "simple"
loss of pruned RNN-T): every lattice factor becomes  c lp_joint + lm_only_scale lp_lm + am_only_scale lp_am  with
c = 1 - lm_only_scale - am_only_scale (include/rnnt.h, rnntSmoothOptions; DESIGN.md §9).  Both 0 is the plain loss.

The keyword-only ``delay_penalty`` is RNNTLoss's: each label factor at frame t gains delay_penalty * ((T_b - 1)/2 - t),
added after the smoothing interpolation (DESIGN.md §10); the loss includes it and the gradients are exact.

The keyword-only ``rnnt_type`` is RNNTLoss's: 'regular' or 'modified' (one symbol per frame, DESIGN.md §11).
"""
import ctypes as C
import math

import torch
from torch.autograd import Function
from torch.nn import Module

from . import warp_rnnt
from ._checks import LengthCheck, check_contiguous, check_dim, check_type

_lib = warp_rnnt.lib()
_P = C.c_void_p
_lib.rnnt_b200_add_joint_loss.restype = C.c_int
_lib.rnnt_b200_add_joint_loss.argtypes = [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P,
                                          warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_forward.restype = C.c_int
_lib.rnnt_b200_add_joint_forward.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P,
                                             warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_backward.restype = C.c_int
_lib.rnnt_b200_add_joint_backward.argtypes = [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P,
                                              warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_backward_ex.restype = C.c_int
_lib.rnnt_b200_add_joint_backward_ex.argtypes = [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float,
                                                 warp_rnnt.rnntGradOptions, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_workspace_size.restype = C.c_int
_lib.rnnt_b200_add_joint_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]


class rnntSmoothOptions(C.Structure):
    """struct rnntSmoothOptions (include/rnnt.h)."""
    _fields_ = [("lm_only_scale", C.c_float), ("am_only_scale", C.c_float)]


_lib.rnnt_b200_add_joint_smoothed_workspace_size.restype = C.c_int
_lib.rnnt_b200_add_joint_smoothed_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int,
                                                             C.POINTER(C.c_size_t)]
_lib.rnnt_b200_add_joint_smoothed_forward.restype = C.c_int
_lib.rnnt_b200_add_joint_smoothed_forward.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int,
                                                      rnntSmoothOptions, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_forward_lat.restype = C.c_int
_lib.rnnt_b200_add_joint_forward_lat.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, rnntSmoothOptions,
                                                 warp_rnnt.rnntLatticeOptions, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_smoothed_backward.restype = C.c_int
_lib.rnnt_b200_add_joint_smoothed_backward.argtypes = [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float,
                                                       warp_rnnt.rnntGradOptions, rnntSmoothOptions, _P,
                                                       warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_forward_topo.restype = C.c_int
_lib.rnnt_b200_add_joint_forward_topo.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int,
                                                  rnntSmoothOptions, warp_rnnt.rnntLatticeOptions, C.c_int, _P,
                                                  warp_rnnt.rnntOptions]
_lib.rnnt_b200_add_joint_backward_topo.restype = C.c_int
_lib.rnnt_b200_add_joint_backward_topo.argtypes = [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float,
                                                   warp_rnnt.rnntGradOptions, rnntSmoothOptions, C.c_int, _P,
                                                   warp_rnnt.rnntOptions]


def smooth_options(lm_only_scale=0.0, am_only_scale=0.0):
    """Checked rnntSmoothOptions, or None when both scales are 0 (the plain entries then run).  Each scale must be
    finite and >= 0, and their sum <= 1, as given (so (0.6, 0.4) is valid although its float32 roundings sum to
    slightly more than 1; the C-ABI allows that one ulp)."""
    lm0, am0 = float(lm_only_scale), float(am_only_scale)
    if not (math.isfinite(lm0) and math.isfinite(am0) and lm0 >= 0.0 and am0 >= 0.0 and lm0 + am0 <= 1.0):
        raise ValueError("lm_only_scale and am_only_scale must be finite, >= 0 and sum to at most 1, got %r, %r"
                         % (lm_only_scale, am_only_scale))
    if lm0 == 0.0 and am0 == 0.0:
        return None
    return rnntSmoothOptions(lm0, am0)


def certify_joint_inputs(trans, pred, labels, lengths, label_lengths, defer=False):
    check_type(labels, torch.int32, "labels")
    check_type(label_lengths, torch.int32, "label_lengths")
    check_type(lengths, torch.int32, "lengths")
    for t, n in ((trans, "trans"), (pred, "pred"), (labels, "labels"), (lengths, "lengths"),
                 (label_lengths, "label_lengths")):
        check_contiguous(t, n)
    check_dim(trans, 3, "trans")
    check_dim(pred, 3, "pred")
    check_dim(labels, 2, "labels")
    if trans.dtype != torch.float32 or pred.dtype != torch.float32:
        raise TypeError("trans and pred must be float32")
    if not (trans.shape[0] == pred.shape[0] == lengths.shape[0] == label_lengths.shape[0]):
        raise ValueError("must have a length and a label length per example.")
    if trans.shape[2] != pred.shape[2]:
        raise ValueError("trans and pred must share the vocabulary dimension")
    check = LengthCheck(lengths, label_lengths, trans.shape[1], pred.shape[1])
    if defer:
        return check
    check.finish()
    return None


def add_joint_call(trans, pred, labels, act_lens, label_lens, costs, dtrans, dpred, blank, scale):
    """Raw call of rnnt_b200_add_joint_loss on CUDA tensors (no checks, no synchronisation)."""
    N, T, V = trans.shape
    U = pred.shape[1]
    n = C.c_size_t(0)
    st = _lib.rnnt_b200_add_joint_workspace_size(T, U, N, V, C.byref(n))
    if st != 0:
        raise ValueError("workspace size: " + warp_rnnt.status_string(st))
    with torch.cuda.device(trans.device):
        ws = torch.empty(n.value, dtype=torch.uint8, device=trans.device)
        opt = warp_rnnt.rnntOptions(loc=1, num_threads=0,
                                    stream=torch.cuda.current_stream(trans.device).cuda_stream,
                                    blank_label=blank, maxT=T, maxU=U, batch_first=True)
        lab = warp_rnnt._labels_ptr(labels)
        st = _lib.rnnt_b200_add_joint_loss(trans.data_ptr(), pred.data_ptr(),
                                           dtrans.data_ptr() if dtrans is not None else None,
                                           dpred.data_ptr() if dpred is not None else None,
                                           lab, label_lens.data_ptr(), act_lens.data_ptr(), V, N,
                                           costs.data_ptr(), scale, ws.data_ptr(), opt)
    if st != 0:
        raise RuntimeError("rnnt_b200_add_joint_loss failed: " + warp_rnnt.status_string(st))
    return ws


def _joint_opts(trans, pred, blank):
    return warp_rnnt.rnntOptions(loc=1, num_threads=0,
                                 stream=torch.cuda.current_stream(trans.device).cuda_stream,
                                 blank_label=blank, maxT=trans.shape[1], maxU=pred.shape[1], batch_first=True)


_lab_ptr = warp_rnnt._labels_ptr   # cached per-device stand-in when there are no labels (U == 1)


def joint_forward_call(trans, pred, labels, act_lens, label_lens, costs, prepare_backward, blank, smooth, lattice=None,
                       topo=warp_rnnt.RNNT_B200_RNNT_REGULAR):
    """The forward half on CUDA tensors (no checks): rnnt_b200_add_joint_forward, or its smoothed form when
    `smooth` (an rnntSmoothOptions) is given, or rnnt_b200_add_joint_forward_lat when `lattice` (an
    rnntLatticeOptions) is given, or rnnt_b200_add_joint_forward_topo for the modified topology `topo`.  Returns
    the workspace the backward half and the ranges read."""
    N, T, V = trans.shape
    U = pred.shape[1]
    n = C.c_size_t(0)
    if smooth is None:
        _lib.rnnt_b200_add_joint_workspace_size(T, U, N, V, C.byref(n))
    else:
        _lib.rnnt_b200_add_joint_smoothed_workspace_size(T, U, N, V, C.byref(n))
    ws = torch.empty(n.value, dtype=torch.uint8, device=trans.device)
    args = (trans.data_ptr(), pred.data_ptr(), _lab_ptr(labels), label_lens.data_ptr(), act_lens.data_ptr(), V, N,
            costs.data_ptr(), 1 if prepare_backward else 0)
    tail = (ws.data_ptr(), _joint_opts(trans, pred, blank))
    if topo != warp_rnnt.RNNT_B200_RNNT_REGULAR:
        st = _lib.rnnt_b200_add_joint_forward_topo(*args, smooth if smooth is not None else rnntSmoothOptions(),
                                                   lattice if lattice is not None else warp_rnnt.rnntLatticeOptions(),
                                                   topo, *tail)
    elif lattice is not None:
        st = _lib.rnnt_b200_add_joint_forward_lat(*args, smooth if smooth is not None else rnntSmoothOptions(),
                                                  lattice, *tail)
    elif smooth is None:
        st = _lib.rnnt_b200_add_joint_forward(*args, *tail)
    else:
        st = _lib.rnnt_b200_add_joint_smoothed_forward(*args, smooth, *tail)
    if st != 0:
        raise RuntimeError("rnnt_b200_add_joint_forward failed: " + warp_rnnt.status_string(st))
    return ws


def check_joint_call(trans, pred, labels, act_lens, label_lens, reduction, fastemit_lambda, lm_only_scale,
                     am_only_scale):
    """Every argument rule of a joint call, before any device work but the delay penalty's (lattice_options):
    (gradient options, smoothing options, deferred length check)."""
    gopt = warp_rnnt.grad_options(fastemit_lambda)   # ValueError before any device work
    if gopt is not None:
        gopt.clamp = 0.0                              # the joint entry accepts no clamp at all
    smooth = smooth_options(lm_only_scale, am_only_scale)
    length_check = certify_joint_inputs(trans, pred, labels, act_lens, label_lens, defer=True)
    if not trans.is_cuda:
        raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only")
    warp_rnnt.require_same_device(trans, pred=pred, labels=labels, act_lens=act_lens, label_lens=label_lens)
    if reduction not in ('none', 'sum', 'mean'):
        raise ValueError("reduction must be 'none', 'sum' or 'mean'")
    return gopt, smooth, length_check


class _AddJointRNNT(Function):
    """forward: factor exponentials, S = Ef.Eg^T, alpha/beta lattices, costs.  backward: weights +
    the two factor-gradient contractions with grad_output[b] and the reduction factor folded in."""

    @staticmethod
    def forward(ctx, trans, pred, labels, act_lens, label_lens, blank, reduction, fastemit_lambda=0.0,
                lm_only_scale=0.0, am_only_scale=0.0, delay_penalty=0.0, rnnt_type='regular'):
        lattice = warp_rnnt.lattice_options(delay_penalty)   # ValueError before any device work
        topo = warp_rnnt.rnnt_type_code(rnnt_type)
        gopt, smooth, length_check = check_joint_call(trans, pred, labels, act_lens, label_lens, reduction,
                                                      fastemit_lambda, lm_only_scale, am_only_scale)
        N = trans.shape[0]
        length_check.guard_labels(labels, N)
        need = trans.requires_grad or pred.requires_grad
        costs = torch.empty(N, dtype=torch.float32, device=trans.device)
        with torch.cuda.device(trans.device):
            ws = joint_forward_call(trans, pred, labels, act_lens, label_lens, costs, need, blank, smooth, lattice,
                                    topo)
        length_check.finish()   # the reference's length test, waited for with the kernels already queued
        if need:
            ctx.save_for_backward(trans, pred, labels, act_lens, label_lens)
            ctx.ws, ctx.blank, ctx.gopt, ctx.smooth, ctx.topo = ws, blank, gopt, smooth, topo
            ctx.scale = 1.0 / N if reduction == 'mean' else 1.0
        if reduction in ('sum', 'mean'):
            costs = costs.sum().unsqueeze_(-1)
            if reduction == 'mean':
                costs /= N
        return costs

    @staticmethod
    def backward(ctx, grad_output):
        trans, pred, labels, act_lens, label_lens = ctx.saved_tensors
        N, T, V = trans.shape
        g = grad_output.reshape(-1).to(device=trans.device, dtype=torch.float32)
        g = g.expand(N).contiguous() if g.numel() == 1 else g.contiguous()
        dtrans, dpred = torch.empty_like(trans), torch.empty_like(pred)
        with torch.cuda.device(trans.device):
            args = (trans.data_ptr(), pred.data_ptr(), dtrans.data_ptr(), dpred.data_ptr(), _lab_ptr(labels),
                    label_lens.data_ptr(), act_lens.data_ptr(), V, N, g.data_ptr(), ctx.scale)
            tail = (ctx.ws.data_ptr(), _joint_opts(trans, pred, ctx.blank))
            if ctx.topo != warp_rnnt.RNNT_B200_RNNT_REGULAR:
                st = _lib.rnnt_b200_add_joint_backward_topo(
                    *args, warp_rnnt.rnntGradOptions() if ctx.gopt is None else ctx.gopt,
                    rnntSmoothOptions() if ctx.smooth is None else ctx.smooth, ctx.topo, *tail)
            elif ctx.smooth is not None:
                gopt = warp_rnnt.rnntGradOptions() if ctx.gopt is None else ctx.gopt
                st = _lib.rnnt_b200_add_joint_smoothed_backward(*args, gopt, ctx.smooth, *tail)
            elif ctx.gopt is not None:
                st = _lib.rnnt_b200_add_joint_backward_ex(*args, ctx.gopt, *tail)
            else:
                st = _lib.rnnt_b200_add_joint_backward(*args, *tail)
        if st != 0:
            raise RuntimeError("rnnt_b200_add_joint_backward failed: " + warp_rnnt.status_string(st))
        return dtrans, dpred, None, None, None, None, None, None, None, None, None, None


def _no_clamp(clamp):
    if clamp is not None:
        raise ValueError("clamp is not available for the additive joint: its factor gradients are contractions "
                         "over the lattice and never form the per-logit gradient that clamp clips")


def add_joint_rnnt_loss(trans, pred, labels, act_lens, label_lens, blank=0, reduction='mean', *,
                        fastemit_lambda=0.0, clamp=None, lm_only_scale=0.0, am_only_scale=0.0, delay_penalty=0.0,
                        rnnt_type='regular'):
    """fastemit_lambda: as rnnt_loss (the gradient is then not the gradient of the returned loss).
    lm_only_scale, am_only_scale: the smoothed loss (module docstring); both 0 is the plain loss.
    delay_penalty: as rnnt_loss, added after the smoothing (module docstring).  rnnt_type: as rnnt_loss."""
    _no_clamp(clamp)
    return _AddJointRNNT.apply(trans, pred, labels, act_lens, label_lens, blank, reduction, fastemit_lambda,
                               lm_only_scale, am_only_scale, delay_penalty, rnnt_type)


class AddJointRNNTLoss(Module):
    def __init__(self, blank=0, reduction='mean', *, fastemit_lambda=0.0, clamp=None, lm_only_scale=0.0,
                 am_only_scale=0.0, delay_penalty=0.0, rnnt_type='regular'):
        super().__init__()
        _no_clamp(clamp)
        warp_rnnt.grad_options(fastemit_lambda)
        smooth_options(lm_only_scale, am_only_scale)
        warp_rnnt.lattice_options(delay_penalty)
        warp_rnnt.rnnt_type_code(rnnt_type)
        self.blank, self.reduction, self.fastemit_lambda = blank, reduction, fastemit_lambda
        self.lm_only_scale, self.am_only_scale = lm_only_scale, am_only_scale
        self.delay_penalty, self.rnnt_type = delay_penalty, rnnt_type

    def forward(self, trans, pred, labels, act_lens, label_lens):
        return _AddJointRNNT.apply(trans, pred, labels, act_lens, label_lens, self.blank, self.reduction,
                                   self.fastemit_lambda, self.lm_only_scale, self.am_only_scale, self.delay_penalty,
                                   self.rnnt_type)
