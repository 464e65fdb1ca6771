"""fp64 CPU reference of the RNN-T loss, gradient and forced alignment on caller-supplied factors (DESIGN.md §13,
include/rnnt.h rnnt_b200_lattice_forward), for the tests.

Factors in k2's orientation: px [N, S, T] (px[b, s, t] = lp_y(t, s)), py [N, S+1, T] (py[b, s, t] = lp_blank(t, s)).
An utterance is T_b = clip(act_lens[b], 1, T) frames and U_b = clip(label_lens[b] + 1, 1, S + 1) contexts, as the
library clamps them; its lattice is lpb = py[b].T[:T_b, :U_b], lpy = px[b].T[:T_b, :U_b - 1], with +inf read as NaN.
The recursions are the existing references': pruned_reference.lattice (regular), modified_reference.lattice /
occupancies (modified), align_reference.align_factors (alignment).  k2's constrained transducer (a label emitted at
frame t is followed by the blank of the next context on the same frame) is enumerated from its definition by
constrained_brute_force.  Test infrastructure only.
"""
import itertools

import numpy as np

import align_reference as ar
import modified_reference as mr
import pruned_reference as pr

NEG = -np.inf


def extents(act_lens, label_lens, T, S):
    """(T_b [N], U_b [N]) after the library's clamps."""
    Tb = np.clip(np.asarray(act_lens, np.int64), 1, T)
    Ub = np.clip(np.asarray(label_lens, np.int64) + 1, 1, S + 1)
    return Tb, Ub


def utterance_factors(px_b, py_b, Tb, Ub):
    """(lpb [T_b, U_b], lpy [T_b, U_b - 1]) of one utterance, float64, +inf as NaN."""
    lpb = np.array(py_b[:Ub, :Tb], np.float64).T.copy()
    lpy = np.array(px_b[:Ub - 1, :Tb], np.float64).T.copy()
    for a in (lpb, lpy):
        a[a == np.inf] = np.nan
    return lpb, lpy


def regular_occupancies(alpha, beta, lpb, lpy, ll):
    """(e_b [T, U], e_y [T, U - 1]) of a regular lattice (pruned_reference.lattice's alpha, beta); zeros without a
    path.  The blank of the last frame exists only at u = U - 1."""
    T, U = lpb.shape
    if ll == NEG:
        return np.zeros((T, U)), np.zeros((T, U - 1))
    e_b = np.zeros((T, U))
    e_b[:T - 1] = np.exp(alpha[:T - 1] + lpb[:T - 1] + beta[1:] - ll)
    e_b[T - 1, U - 1] = np.exp(alpha[T - 1, U - 1] + lpb[T - 1, U - 1] - ll)
    e_y = np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - ll)
    return e_b, e_y


def utterance_loss(lpb, lpy, modified=False):
    """(cost, e_b, e_y) of one utterance's factors."""
    if modified:
        alpha, beta, ll = mr.lattice(lpb, lpy)
        e_b, e_y = mr.occupancies(alpha, beta, lpb, lpy, ll)
    else:
        alpha, beta, ll = pr.lattice(lpb, lpy)
        e_b, e_y = regular_occupancies(alpha, beta, lpb, lpy, ll)
    return -ll, e_b, e_y


def loss(px, py, act_lens, label_lens, modified=False):
    """(costs [N], px_grad [N, S, T], py_grad [N, S+1, T]) in float64: d cost[b] / d px, d cost[b] / d py, zero on
    padding and without a path."""
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    N, S1, T = py.shape
    Tb, Ub = extents(act_lens, label_lens, T, S1 - 1)
    costs = np.zeros(N)
    gx, gy = np.zeros(px.shape), np.zeros(py.shape)
    for b in range(N):
        lpb, lpy = utterance_factors(px[b], py[b], Tb[b], Ub[b])
        costs[b], e_b, e_y = utterance_loss(lpb, lpy, modified)
        gy[b, :Ub[b], :Tb[b]] = -e_b.T
        gx[b, :Ub[b] - 1, :Tb[b]] = -e_y.T
    return costs, gx, gy


def align(px, py, act_lens, label_lens, modified=False):
    """(scores [N], frames [N, S]) of the best alignments, align_reference's contract."""
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    N, S1, T = py.shape
    Tb, Ub = extents(act_lens, label_lens, T, S1 - 1)
    scores = np.zeros(N)
    frames = np.full((N, S1 - 1), -1, np.int64)
    for b in range(N):
        lpb, lpy = utterance_factors(px[b], py[b], Tb[b], Ub[b])
        scores[b], f = ar.align_factors(lpb, lpy, modified)
        frames[b, :Ub[b] - 1] = f
    return scores, frames


def factors_from_logits(logits, labels, blank=0):
    """k2-oriented (px [N, U-1, T], py [N, U, T]) gathered from log_softmax(logits [N, T, U, V])."""
    lp = pr.log_softmax(np.asarray(logits, np.float64))
    N, T, U, _ = lp.shape
    py = lp[..., blank].transpose(0, 2, 1).copy()
    px = np.zeros((N, U - 1, T))
    for b in range(N):
        for u in range(U - 1):
            px[b, u] = lp[b, :, u, labels[b, u]]
    return px, py


def brute_force(lpb, lpy, modified=False):
    """-(logsumexp over every path) of one utterance, by enumeration (align_reference.all_alignments); +inf
    without a path."""
    return -ar.brute_force(lpb, lpy, modified)[3]


def constrained_brute_force(lpb, lpy):
    """Cost of k2's constrained transducer by enumeration: every frame emits either the blank of its context, or
    the label of its context followed by the blank of the next context on the same frame; the frames that emit
    labels strictly increase.  +inf without a path."""
    T, U = lpb.shape
    scores = []
    for ts in itertools.combinations(range(T), U - 1):
        s, u = 0.0, 0
        for t in range(T):
            if u < U - 1 and ts[u] == t:
                s += lpy[t, u] + lpb[t, u + 1]
                u += 1
            else:
                s += lpb[t, u]
        scores.append(s)
    return -np.logaddexp.reduce(np.array(scores)) if scores else np.inf


def torch_ll(lpb, lpy, modified=False):
    """Differentiable log-likelihood of torch fp64 factors lpb [T, U], lpy [T, U - 1] (finite factors)."""
    import torch
    if modified:
        return mr._torch_ll(lpb, lpy)
    T, U = lpb.shape
    alpha = [[None] * U for _ in range(T)]
    for t in range(T):
        for u in range(U):
            terms = []
            if t > 0:
                terms.append(alpha[t - 1][u] + lpb[t - 1, u])
            if u > 0:
                terms.append(alpha[t][u - 1] + lpy[t, u - 1])
            alpha[t][u] = torch.logsumexp(torch.stack(terms), 0) if terms else torch.zeros((), dtype=lpb.dtype)
    return alpha[T - 1][U - 1] + lpb[T - 1, U - 1]
