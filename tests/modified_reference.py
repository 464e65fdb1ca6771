"""fp64 CPU reference of the modified (one symbol per frame) transducer (DESIGN.md §11, include/rnnt.h
RNNT_B200_RNNT_MODIFIED), for the tests.

Every frame takes exactly one transition, a blank (u stays) or the label y_u (u + 1), both to the next frame:
    alpha(0,0) = 0,  alpha(t,u) = lse(alpha(t-1,u) + lp_blank(t-1,u), alpha(t-1,u-1) + lp_y(t-1,u-1))
    ll = lse(alpha(T-1,U-1) + lp_blank(T-1,U-1), alpha(T-1,U-2) + lp_y(T-1,U-2))    (the virtual cell (T, U-1))
    beta(T,U-1) = 0, beta(T,u) = log zero otherwise,  beta(t,u) = lse(lp_blank(t,u) + beta(t+1,u), lp_y(t,u) + beta(t+1,u+1))
The references compose the existing ones: the factors of pruned_reference (dense: R = maxU, ranges == 0) with the
penalty of delay_reference, the factors of smoothed_reference for the joint, and the window rule of
pruned_reference.prune_ranges.  No path (U_b - 1 > T_b, or pruned windows that leave none): cost +inf, zero gradient.
Test infrastructure only.
"""
import contextlib
import itertools

import numpy as np

import delay_reference as dr
import pruned_reference as pr
import smoothed_reference as sr

NEG = -np.inf


def lattice(lpb, lpy):
    """(alpha [T, U], beta [T + 1, U] with the virtual row T, ll) of the modified lattice; lpb [T, U],
    lpy [T, U - 1]."""
    T, U = lpb.shape
    alpha = np.full((T, U), NEG)
    alpha[0, 0] = 0.0
    for t in range(1, T):
        for u in range(U):
            a = alpha[t - 1, u] + lpb[t - 1, u]
            b = alpha[t - 1, u - 1] + lpy[t - 1, u - 1] if u > 0 else NEG
            alpha[t, u] = np.logaddexp(a, b)
    last = alpha[T - 1, U - 2] + lpy[T - 1, U - 2] if U > 1 else NEG
    ll = np.logaddexp(alpha[T - 1, U - 1] + lpb[T - 1, U - 1], last)
    beta = np.full((T + 1, U), NEG)
    beta[T, U - 1] = 0.0
    for t in range(T - 1, -1, -1):
        for u in range(U):
            b = lpy[t, u] + beta[t + 1, u + 1] if u < U - 1 else NEG
            beta[t, u] = np.logaddexp(lpb[t, u] + beta[t + 1, u], b)
    return alpha, beta, ll


def occupancies(alpha, beta, lpb, lpy, ll):
    """(e_b [T, U], e_y [T, U - 1]): the blank and label transition occupancies of a modified lattice; zeros when
    it has no path."""
    T, U = lpb.shape
    if ll == NEG:
        return np.zeros((T, U)), np.zeros((T, U - 1))
    e_b = np.exp(alpha + lpb + beta[1:] - ll)
    e_y = np.exp(alpha[:, :U - 1] + lpy + beta[1:, 1:] - ll)
    return e_b, e_y


def loss(logits, labels, act_lens, label_lens, ranges=None, blank=0, delay_penalty=0.0, fastemit_lambda=0.0,
         clamp=-1.0):
    """(costs [N], gradient [N, maxT, R, V]) in float64.  ranges None: the dense loss (R must be maxU).  FastEmit,
    clamp and the delay penalty as delay_reference.loss, on the modified lattice."""
    logits = np.asarray(logits, dtype=np.float64)
    N, maxT, R, V = logits.shape
    labels = np.asarray(labels).reshape(N, -1)
    ranges = np.zeros((N, maxT), np.int64) if ranges is None else np.asarray(ranges, np.int64)
    lam, fe = float(delay_penalty), float(fastemit_lambda)
    costs = np.zeros(N)
    grads = np.zeros_like(logits)
    for b in range(N):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lp = pr.log_softmax(logits[b])
        lpb, lpy, cell = pr.pruned_factors(lp, labels[b], ranges[b], T, U, blank)
        lpy = lpy + dr.penalty(T, U - 1, lam)
        alpha, beta, ll = lattice(lpb, lpy)
        if ll == NEG:
            costs[b] = np.inf
            continue
        costs[b] = -ll
        e_b, e_y = occupancies(alpha, beta, lpb, lpy, ll)
        for t in range(T):
            for s in range(R):
                u = cell[t, s]
                if u < 0:
                    continue
                p = np.exp(lp[t, s])
                ey = e_y[t, u] if u < U - 1 else 0.0
                g = p * (np.exp(alpha[t, u] + beta[t, u] - ll) + fe * ey)
                g[blank] -= e_b[t, u]
                if u < U - 1:
                    g[labels[b, u]] -= (1.0 + fe) * ey
                grads[b, t, s] = np.clip(g, -clamp, clamp) if clamp > 0 else g
    return costs, grads


def dense_loss(acts, labels, act_lens, label_lens, blank=0, delay_penalty=0.0, fastemit_lambda=0.0, clamp=-1.0):
    """loss() of dense logits [N, T, U, V]."""
    return loss(acts, labels, act_lens, label_lens, None, blank, delay_penalty, fastemit_lambda, clamp)


def brute_force(acts, labels, T, U, blank=0, delay_penalty=0.0):
    """Cost of one utterance's logits [T, U, V] by summing over every path: the strictly increasing frames
    t_1 < ... < t_{U-1} that emit the labels; every other frame emits a blank.  +inf when there is none."""
    lp = pr.log_softmax(np.asarray(acts, np.float64)[:T, :U])
    lam = float(delay_penalty)
    scores = []
    for ts in itertools.combinations(range(T), U - 1):
        s, u = 0.0, 0
        for t in range(T):
            if u < U - 1 and ts[u] == t:
                s += lp[t, u, labels[u]] + lam * ((T - 1) / 2.0 - t)
                u += 1
            else:
                s += lp[t, u, blank]
        scores.append(s)
    return -np.logaddexp.reduce(np.array(scores)) if scores else np.inf


def _torch_ll(lpb, lpy):
    """Modified log-likelihood (torch, differentiable); lpb [T, U], lpy [T, U - 1]."""
    import torch
    T, U = lpb.shape
    neg = torch.tensor(NEG, dtype=lpb.dtype)
    if U - 1 > T:
        return neg   # no path: a constant, so that it sends no (NaN) gradient into factors other costs share
    row = [torch.zeros((), dtype=lpb.dtype)] + [neg] * (U - 1)
    for t in range(1, T + 1):
        # after t frames only u <= t is reached; those cells stay the constant log zero, as logaddexp of two log
        # zeros would send NaN gradients back
        nxt = []
        for u in range(U):
            if u > t:
                nxt.append(neg)
                continue
            x = row[u] + lpb[t - 1, u] if u < t else neg
            z = row[u - 1] + lpy[t - 1, u - 1] if u > 0 else neg
            nxt.append(torch.logaddexp(x, z))
        row = nxt
    return row[U - 1]   # alpha of the virtual cell (T, U - 1)


@contextlib.contextmanager
def modified_lattice(delay_penalty=0.0):
    """Within the block, smoothed_reference's torch lattice is the modified one, with the penalty added to the
    label factors it is given (after smoothing and FastEmit, as delay_reference.penalised_lattice)."""
    import torch
    plain = sr._torch_ll
    lam = float(delay_penalty)

    def ll(lpb, lpy):
        T, n = lpy.shape
        return _torch_ll(lpb, lpy + torch.tensor(dr.penalty(T, n, lam), dtype=lpy.dtype))

    sr._torch_ll = ll
    try:
        yield
    finally:
        sr._torch_ll = plain


def torch_dense_costs(acts, labels, act_lens, label_lens, blank=0, delay_penalty=0.0):
    """[N] modified costs of torch fp64 logits [N, T, U, V], differentiable."""
    with modified_lattice(delay_penalty):
        import torch
        out = []
        for b in range(acts.shape[0]):
            T, U = int(act_lens[b]), int(label_lens[b]) + 1
            lp = torch.log_softmax(acts[b, :T, :U], dim=-1)
            y = torch.as_tensor(np.asarray(labels[b][:U - 1], np.int64))
            lpy = lp[:, torch.arange(U - 1), y] if U > 1 else torch.zeros((T, 0), dtype=acts.dtype)
            out.append(-sr._torch_ll(lp[:, :, blank], lpy))
        return torch.stack(out)


def joint_costs(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    return np.array([-lattice(lpb, lpy)[2] for lpb, lpy in
                     dr.joint_factors(trans, pred, labels, act_lens, label_lens, lm, am, blank, delay_penalty)])


def joint_reference(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0,
                    fastemit_lambda=0.0, scale=None):
    """smoothed_reference.reference on the modified lattice: (costs [N], dF [N,T,V], dG [N,U,V]) in float64.  An
    utterance without a path has cost +inf and contributes no gradient."""
    with modified_lattice(delay_penalty):
        return sr.reference(trans, pred, labels, act_lens, label_lens, lm, am, blank, fastemit_lambda, scale)


def joint_occupancies(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    """Per utterance (e_b, e_y) of the modified joint lattice, the input of pruned_reference.prune_ranges."""
    out = []
    for lpb, lpy in dr.joint_factors(trans, pred, labels, act_lens, label_lens, lm, am, blank, delay_penalty):
        alpha, beta, ll = lattice(lpb, lpy)
        out.append(occupancies(alpha, beta, lpb, lpy, ll))
    return out


def prune_ranges(trans, pred, labels, act_lens, label_lens, maxT, R, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    """[N, maxT] window starts of a modified joint workspace (steps 1-3 of DESIGN.md §8 on the modified
    occupancies) and the smallest score margin, as pruned_reference.prune_ranges."""
    return pr.prune_ranges(joint_occupancies(trans, pred, labels, act_lens, label_lens, lm, am, blank,
                                             delay_penalty), maxT, R)
