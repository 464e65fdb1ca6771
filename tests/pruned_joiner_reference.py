"""fp64 torch reference of the pruned fused joiner (DESIGN.md §15, include/rnnt.h rnnt_b200_pruned_joiner_forward /
_backward), for the tests: the fused joiner's reference (tests/joiner_reference.py) with its factors masked to the
cells a valid window row covers.

    covered[b, t, u]  = some r < R has u = ranges[b, t] + r, with t < T_b and 0 <= u <= S_b
    px, py            = jr.log_probs(...) on covered cells, -inf elsewhere
    gradients(dpx, dpy) = jr.gradients(dpx masked, dpy masked)       (masked: 0 off the covered cells, NaN included)

Test infrastructure only.
"""
import torch

import joiner_reference as jr


def covered(ranges, s_range, act_lens, label_lens, T, U):
    """[N, T, U] bool: the cells a valid row (b, t, r) stands for.  Window starts are widened to int64 first, so any
    int32 start is well defined."""
    N = ranges.shape[0]
    u = ranges.long()[:, :, None] + torch.arange(s_range, device=ranges.device)       # [N, T, R]
    inside = (u >= 0) & (u < U)
    b, t, r = inside.nonzero(as_tuple=True)
    cov = torch.zeros(N, T, U, dtype=torch.bool, device=ranges.device)
    cov[b, t, u[b, t, r]] = True
    cell, _ = jr.masks(act_lens, label_lens, T, U)
    return cov & cell


def factor_masks(ranges, s_range, act_lens, label_lens, T, U):
    """(mx [N, U-1, T], my [N, U, T]): where px and py of the pruned lattice are not -inf."""
    cov = covered(ranges, s_range, act_lens, label_lens, T, U)
    _, lab = jr.masks(act_lens, label_lens, T, U)
    return (cov[..., :U - 1] & lab).permute(0, 2, 1), cov.permute(0, 2, 1)


def log_probs(h, weight, bias, labels, act_lens, label_lens, ranges, s_range, blank=0):
    """fp64 (px [N, U-1, T], py [N, U, T]) of the pruned lattice, from the dense h [N, T, U, H]."""
    N, T, U, _ = h.shape
    px, py = jr.log_probs(h, weight, bias, labels, act_lens, label_lens, blank)
    mx, my = factor_masks(ranges, s_range, act_lens, label_lens, T, U)
    return px.masked_fill(~mx, -float('inf')), py.masked_fill(~my, -float('inf'))


def masked_incoming(dpx, dpy, ranges, s_range, act_lens, label_lens):
    """dpx, dpy as fp64 with every element off the covered cells (NaN included) set to 0."""
    N, U, T = dpy.shape
    mx, my = factor_masks(ranges, s_range, act_lens, label_lens, T, U)
    zx, zy = torch.zeros((), dtype=torch.float64, device=dpy.device), torch.zeros((), dtype=torch.float64,
                                                                                  device=dpy.device)
    return torch.where(mx, dpx.double(), zx), torch.where(my, dpy.double(), zy)


def gradients(h, weight, bias, labels, act_lens, label_lens, dpx, dpy, ranges, s_range, activation, blank=0):
    """fp64 (d_enc, d_pred, d_weight, d_bias): the dense gradients of the masked incoming gradients."""
    gx, gy = masked_incoming(dpx, dpy, ranges, s_range, act_lens, label_lens)
    return jr.gradients(h, weight, bias, labels, act_lens, label_lens, gx, gy, activation, blank)
