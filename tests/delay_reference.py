"""fp64 CPU reference of the delay penalty (DESIGN.md §10, include/rnnt.h rnntLatticeOptions), for the tests.

With lambda = delay_penalty and T_b the utterance's frame count, every label factor of a valid cell gains
    pen(t) = lambda ((T_b - 1)/2 - t)
and nothing else changes.  The references below compose the existing ones rather than fork them:
  loss()           the dense or pruned loss of logits [N, maxT, R, V] (dense: R = maxU and ranges == 0), from
                   pruned_reference.pruned_factors + the penalty + pruned_reference.lattice; the gradient is the
                   dense formula with the penalised occupancies and, for FastEmit, the unpenalised p_y.
  joint_factors()  smoothed_reference.factors plus the penalty (the penalty comes after the smoothing).
  joint_reference() costs and factor gradients from smoothed_reference.torch_costs under torch fp64 autograd, with
                   the penalty added to the label factors just before the lattice (penalised_lattice()).
  brute_force()    the cost by enumerating every path, with the penalty written per path.
Test infrastructure only.
"""
import contextlib
import itertools

import numpy as np

import pruned_reference as pr
import smoothed_reference as sr


def penalty(T, n, lam):
    """[T, n] penalty of the label factors of an utterance with T frames (n = U_b - 1 label columns)."""
    return np.broadcast_to(lam * ((T - 1) / 2.0 - np.arange(T, dtype=np.float64))[:, None], (T, n))


def loss(logits, labels, act_lens, label_lens, ranges=None, blank=0, delay_penalty=0.0, fastemit_lambda=0.0,
         clamp=-1.0):
    """(costs [N], gradient [N, maxT, R, V]) in float64.  ranges None: the dense loss (R must be maxU)."""
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
        lpy = lpy + penalty(T, U - 1, lam)          # log zero stays log zero
        alpha, beta, ll = pr.lattice(lpb, lpy)
        if ll == -np.inf:
            costs[b] = np.inf
            continue
        costs[b] = -ll
        for t in range(T):
            for s in range(R):
                u = cell[t, s]
                if u < 0:
                    continue
                p = np.exp(lp[t, s])
                occ = np.exp(alpha[t, u] + beta[t, u] - ll)
                if t < T - 1:
                    e_b = np.exp(alpha[t, u] + lpb[t, u] + beta[t + 1, u] - ll)
                else:
                    e_b = np.exp(alpha[t, u] + lpb[t, u] - ll) if u == U - 1 else 0.0
                e_y = np.exp(alpha[t, u] + lpy[t, u] + beta[t, u + 1] - ll) if u < U - 1 else 0.0
                g = p * (occ + fe * e_y)
                g[blank] -= e_b
                if u < U - 1:
                    g[labels[b, u]] -= (1.0 + fe) * e_y
                grads[b, t, s] = np.clip(g, -clamp, clamp) if clamp > 0 else g
    return costs, grads


def dense_loss(acts, labels, act_lens, label_lens, blank=0, delay_penalty=0.0, fastemit_lambda=0.0, clamp=-1.0):
    """loss() of dense logits [N, T, U, V]."""
    return loss(acts, labels, act_lens, label_lens, None, blank, delay_penalty, fastemit_lambda, clamp)


def brute_force(acts, labels, T, U, blank=0, delay_penalty=0.0):
    """Cost of one utterance's logits [T, U, V] by summing over every path: a path is the frames t_1 <= ... <=
    t_{U-1} at which the labels are emitted; each frame ends with one blank.  The penalty is added per path as
    lambda sum_i ((T - 1)/2 - t_i)."""
    lp = pr.log_softmax(np.asarray(acts, np.float64)[:T, :U])
    lam = float(delay_penalty)
    scores = []
    for ts in itertools.combinations_with_replacement(range(T), U - 1):
        s = 0.0
        for i, t in enumerate(ts):
            s += lp[t, i, labels[i]] + lam * ((T - 1) / 2.0 - t)
        for t in range(T):
            u = sum(1 for x in ts if x <= t)
            s += lp[t, u, blank]
        scores.append(s)
    return -np.logaddexp.reduce(np.array(scores))


def joint_factors(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    """smoothed_reference.factors with the penalty on the label factors."""
    return [(lpb, lpy + penalty(lpb.shape[0], lpy.shape[1], float(delay_penalty)))
            for lpb, lpy in sr.factors(trans, pred, labels, act_lens, label_lens, lm, am, blank)]


def joint_costs(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    return np.array([-pr.lattice(lpb, lpy)[2] for lpb, lpy in
                     joint_factors(trans, pred, labels, act_lens, label_lens, lm, am, blank, delay_penalty)])


def joint_occupancies(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0):
    """As smoothed_reference.smoothed_occupancies, on the penalised lattice (pruned_reference.prune_ranges input)."""
    out = []
    for lpb, lpy in joint_factors(trans, pred, labels, act_lens, label_lens, lm, am, blank, delay_penalty):
        T, U = lpb.shape
        alpha, beta, ll = pr.lattice(lpb, lpy)
        e_b = np.zeros((T, U))
        e_b[:T - 1] = np.exp(alpha[:T - 1] + lpb[:T - 1] + beta[1:] - ll)
        e_y = np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - ll)
        out.append((e_b, e_y))
    return out


@contextlib.contextmanager
def penalised_lattice(delay_penalty):
    """Within the block, smoothed_reference's torch lattice adds the penalty to the label factors it is given.
    torch_costs applies FastEmit to the label factors before calling it, so the penalty comes after the smoothing
    and FastEmit scales the gradient of the penalised factor, as the library does."""
    import torch
    plain = sr._torch_ll
    lam = float(delay_penalty)

    def ll(lpb, lpy):
        T, n = lpy.shape
        return plain(lpb, lpy + torch.tensor(penalty(T, n, lam), dtype=lpy.dtype))

    sr._torch_ll = ll
    try:
        yield
    finally:
        sr._torch_ll = plain


def joint_reference(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, delay_penalty=0.0,
                    fastemit_lambda=0.0, scale=None):
    """smoothed_reference.reference on the penalised lattice: (costs [N], dF [N,T,V], dG [N,U,V]) in float64."""
    with penalised_lattice(delay_penalty):
        return sr.reference(trans, pred, labels, act_lens, label_lens, lm, am, blank, fastemit_lambda, scale)


def torch_dense_costs(acts, labels, act_lens, label_lens, blank=0, delay_penalty=0.0):
    """[N] costs of torch fp64 logits [N, T, U, V], differentiable (the lattice of smoothed_reference)."""
    import torch
    out = []
    for b in range(acts.shape[0]):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lp = torch.log_softmax(acts[b, :T, :U], dim=-1)
        y = torch.as_tensor(np.asarray(labels[b][:U - 1], np.int64))
        lpb = lp[:, :, blank]
        lpy = lp[:, torch.arange(U - 1), y] if U > 1 else torch.zeros((T, 0), dtype=acts.dtype)
        with penalised_lattice(delay_penalty):
            out.append(-sr._torch_ll(lpb, lpy))
    return torch.stack(out)
