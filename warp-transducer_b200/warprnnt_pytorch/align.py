"""Forced alignment on the RNN-T lattice (DESIGN.md §12): the highest-scoring path of each utterance and the frame
at which it emits each label - token timestamps, symbol delay, and a check of where a pruned loss's windows lie.

    frames, scores = rnnt_forced_align(logits, labels, act_lens, label_lens)
    # frames [N, U-1] int32: encoder frame of label j (-1 past label_lens[b]); scores [N]: log-probability of the path

The lattice is the loss's (rnnt_loss / pruned_rnnt_loss with the same arguments), without a delay penalty.  Among
equally good partial paths the one that emits its labels earlier wins.  An utterance without a path gets
scores = -inf and frames = -1, one with a NaN logit scores = NaN and frames = -1.
"""
import torch

from . import warp_rnnt
from ._checks import certify_inputs
from .pruned import _check_pruned_inputs


def rnnt_forced_align(acts, labels, act_lens, label_lens, blank=0, *, rnnt_type='regular'):
    """(frames, scores) of the best alignment of acts [N, T, U, V] (raw joint logits, fp32 / fp64 / bf16 / fp16).
    labels, lengths and blank follow rnnt_loss, and so do the input checks and their exceptions.  rnnt_type:
    'regular' (frames non-decreasing) or 'modified' (at most one label per frame: frames strictly increasing).
    frames is [N, U-1] int32, scores [N] float32 (float64 for fp64 logits); natural log, <= 0.  The result carries
    no autograd graph."""
    warp_rnnt.rnnt_type_code(rnnt_type)   # ValueError before any device work
    length_check = certify_inputs(acts, labels, act_lens, label_lens, defer=True)
    if not acts.is_cuda:
        raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only; there is no CPU fallback")
    warp_rnnt.require_same_device(acts, labels=labels, act_lens=act_lens, label_lens=label_lens)
    N, _, U, _ = acts.shape
    length_check.guard_labels(labels, N)
    frames = torch.empty((N, U - 1), dtype=torch.int32, device=acts.device)
    scores = torch.empty(N, dtype=warp_rnnt.costs_dtype(acts), device=acts.device)
    warp_rnnt.gpu_rnnt_align(acts.detach(), labels, act_lens, label_lens, frames, scores, blank, rnnt_type=rnnt_type)
    length_check.finish()
    return frames, scores


def pruned_rnnt_forced_align(logits, labels, act_lens, label_lens, ranges, blank=0, *, rnnt_type='regular'):
    """rnnt_forced_align for pruned logits [N, T, R, V] over the windows ranges [N, T] (pruned_rnnt_loss's inputs
    and checks): the best path through the covered cells.  An utterance whose windows leave no path gets
    scores = -inf and frames = -1.  With R = U and ranges == 0 this is rnnt_forced_align exactly."""
    warp_rnnt.rnnt_type_code(rnnt_type)
    warp_rnnt._dtype_code(logits)
    length_check = _check_pruned_inputs(logits, labels, act_lens, label_lens, ranges)
    N = logits.shape[0]
    U = labels.shape[1] + 1
    length_check.guard_labels(labels, N)
    frames = torch.empty((N, U - 1), dtype=torch.int32, device=logits.device)
    scores = torch.empty(N, dtype=warp_rnnt.costs_dtype(logits), device=logits.device)
    warp_rnnt.gpu_pruned_rnnt_align(logits.detach(), ranges, labels, act_lens, label_lens, frames, scores, blank,
                                    rnnt_type=rnnt_type)
    length_check.finish()
    return frames, scores
