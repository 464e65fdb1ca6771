"""fp64 CPU reference of the smoothed additive joint (DESIGN.md §9, include/rnnt.h rnntSmoothOptions), for the tests.

With f = trans [N,T,V], g = pred [N,U,V], U_b = label_len_b + 1 and c = 1 - lm - am, the factors of a valid cell
(t < T_b, u < U_b) for k in {blank, y_u} (the label only for u < U_b - 1) are

    lp(t,u,k) = c (f[t,k] + g[u,k] - lse(t,u)) + lm (g[u,k] - Lg(u)) + am (f[t,k] + log ug[k] - La(t))

  lse(t,u) = log sum_v exp(f[t,v] + g[u,v]),  Lg(u) = log sum_v exp(g[u,v]),  La(t) = log sum_v exp(f[t,v]) ug[v],
  ug[v]    = (1/M) sum over the M = sum_b U_b valid pred rows of the batch of softmax(g[b,u])[v], plus FLT_MIN.

A term whose scale is exactly 0 is left out.  The cost is -log-likelihood of the standard lattice on these factors
(pruned_reference.lattice).  factors() / costs() are numpy; torch_costs() is the same forward in torch fp64, whose
autograd is the reference gradient (it includes the path through ug).  smoothed_occupancies() feeds
pruned_reference.prune_ranges the windows of the smoothed lattice.  closed_form() gives reference()'s results from
the chain rule written out term by term, one utterance at a time: it never forms [T, U, V] and reaches training
shapes that the autograd reference cannot.
"""
import numpy as np

from pruned_reference import lattice

FLT_MIN = float(np.finfo(np.float32).tiny)


def _lse(x, axis=-1):
    m = x.max(axis=axis, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    return (m + np.log(np.exp(x - m).sum(axis=axis, keepdims=True))).squeeze(axis)


def extents(act_lens, label_lens, T, U):
    return [(min(max(int(a), 1), T), min(max(int(y) + 1, 1), U)) for a, y in zip(act_lens, label_lens)]


def unigram(pred, act_lens, label_lens):
    """ug [V] over the batch's valid pred rows (padded rows are not read)."""
    pred = np.asarray(pred, np.float64)
    ext = extents(act_lens, label_lens, 1 << 30, pred.shape[1])
    rows = np.concatenate([pred[b, :Ub] for b, (_, Ub) in enumerate(ext)])
    p = np.exp(rows - _lse(rows)[:, None])
    return p.mean(axis=0) + FLT_MIN


def factors(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0):
    """Per utterance (lpb [T_b, U_b], lpy [T_b, U_b - 1]) of the smoothed lattice."""
    trans, pred = np.asarray(trans, np.float64), np.asarray(pred, np.float64)
    N, T, V = trans.shape
    U = pred.shape[1]
    c = 1.0 - lm - am
    ug = unigram(pred, act_lens, label_lens) if am != 0.0 else None
    out = []
    for b, (Tb, Ub) in enumerate(extents(act_lens, label_lens, T, U)):
        f, g = trans[b, :Tb], pred[b, :Ub]
        y = np.asarray(labels[b][:Ub - 1], np.int64) if Ub > 1 else np.zeros(0, np.int64)

        def lp(k_cols):
            """[T_b, U_b or U_b-1] factor of column k_cols[u] at (t, u)."""
            n = len(k_cols)
            out_ = np.zeros((Tb, n))
            fk = f[:, k_cols]                       # [Tb, n]
            gk = g[np.arange(n), k_cols][None, :]   # [1, n]
            if c != 0.0:
                lse = _lse(f[:, None, :] + g[None, :n, :])   # [T_b, n]
                out_ = out_ + c * (fk + gk - lse)
            if lm != 0.0:
                out_ = out_ + lm * (gk - _lse(g[:n])[None, :])
            if am != 0.0:
                La = _lse(f + np.log(ug)[None, :])[:, None]
                out_ = out_ + am * (fk + np.log(ug[k_cols])[None, :] - La)
            return out_

        lpb = lp(np.full(Ub, blank, np.int64))
        lpy = lp(y) if Ub > 1 else np.zeros((Tb, 0))
        out.append((lpb, lpy))
    return out


def costs(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0):
    """[N] float64 costs."""
    return np.array([-lattice(lpb, lpy)[2] for lpb, lpy in
                     factors(trans, pred, labels, act_lens, label_lens, lm, am, blank)])


def smoothed_occupancies(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0):
    """As pruned_reference.simple_occupancies, on the smoothed lattice."""
    out = []
    for lpb, lpy in factors(trans, pred, labels, act_lens, label_lens, lm, am, blank):
        T, U = lpb.shape
        alpha, beta, ll = lattice(lpb, lpy)
        e_b = np.zeros((T, U))
        e_b[:T - 1] = np.exp(alpha[:T - 1] + lpb[:T - 1] + beta[1:] - ll)
        e_y = np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - ll)
        out.append((e_b, e_y))
    return out


# ---- torch fp64 forward: autograd is the reference gradient -------------------------------------------------------
def _torch_ll(lpb, lpy):
    """log-likelihood of the lattice (torch, differentiable); lpb [T,U], lpy [T,U-1]."""
    import torch
    T, U = lpb.shape
    neg = torch.tensor(-np.inf, dtype=lpb.dtype)
    prev = [None] * U   # alpha of row t-1
    for t in range(T):
        row = []
        for u in range(U):
            if t == 0 and u == 0:
                a = torch.zeros((), dtype=lpb.dtype)
            else:
                x = prev[u] + lpb[t - 1, u] if t > 0 else neg
                z = row[u - 1] + lpy[t, u - 1] if u > 0 else neg
                a = torch.logaddexp(x, z)
            row.append(a)
        prev = row
    return prev[U - 1] + lpb[T - 1, U - 1]


def torch_costs(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, fastemit_lambda=0.0):
    """[N] costs from torch fp64 tensors trans [N,T,V], pred [N,U,V] (differentiable).  fastemit_lambda > 0 scales
    the gradient of every label factor by 1 + lambda without changing the value (FastEmit)."""
    import torch
    N, T, V = trans.shape
    U = pred.shape[1]
    c = 1.0 - lm - am
    ext = extents(act_lens, label_lens, T, U)
    if am != 0.0:
        rows = torch.cat([pred[b, :Ub] for b, (_, Ub) in enumerate(ext)])
        ug = torch.softmax(rows, dim=-1).mean(dim=0) + FLT_MIN
        lug = torch.log(ug)
    out = []
    for b, (Tb, Ub) in enumerate(ext):
        f, g = trans[b, :Tb], pred[b, :Ub]
        y = torch.as_tensor(np.asarray(labels[b][:Ub - 1], np.int64)) if Ub > 1 else torch.zeros(0, dtype=torch.long)
        lse = torch.logsumexp(f[:, None, :] + g[None, :, :], dim=-1)     # [Tb, Ub]
        Lg = torch.logsumexp(g, dim=-1)
        La = torch.logsumexp(f + lug[None, :], dim=-1) if am != 0.0 else None

        def lp(k, n):
            fk = f[:, k]
            gk = g[torch.arange(n), k][None, :]
            out_ = torch.zeros((Tb, n), dtype=f.dtype)
            if c != 0.0:
                out_ = out_ + c * (fk + gk - lse[:, :n])
            if lm != 0.0:
                out_ = out_ + lm * (gk - Lg[None, :n])
            if am != 0.0:
                out_ = out_ + am * (fk + lug[k][None, :] - La[:, None])
            return out_

        lpb = lp(torch.full((Ub,), blank, dtype=torch.long), Ub)
        lpy = lp(y, Ub - 1) if Ub > 1 else torch.zeros((Tb, 0), dtype=f.dtype)
        if fastemit_lambda:
            lpy = lpy + fastemit_lambda * (lpy - lpy.detach())
        out.append(-_torch_ll(lpb, lpy))
    return torch.stack(out)


def reference(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, fastemit_lambda=0.0, scale=None):
    """(costs [N], dF [N,T,V], dG [N,U,V]) in float64; the gradient of sum_b scale[b] cost_b (scale default 1)."""
    import torch
    f = torch.tensor(np.asarray(trans, np.float64), requires_grad=True)
    g = torch.tensor(np.asarray(pred, np.float64), requires_grad=True)
    c = torch_costs(f, g, labels, act_lens, label_lens, lm, am, blank, fastemit_lambda)
    w = torch.ones_like(c) if scale is None else torch.as_tensor(np.asarray(scale, np.float64))
    (c * w).sum().backward()
    grad = lambda x: np.zeros(x.shape) if x.grad is None else x.grad.numpy()   # noqa: E731  (lm = 1: no trans path)
    return c.detach().numpy(), grad(f), grad(g)


# ---- closed form: the same costs and gradients without autograd and without any [T, U, V] array ------------------
def _exp_rows(x):
    """(E = exp(x - m), m) per row, m the row max (0 for an all -inf row)."""
    m = x.max(axis=1)
    m = np.where(np.isfinite(m), m, 0.0)
    return np.exp(x - m[:, None]), m


def closed_form(trans, pred, labels, act_lens, label_lens, lm=0.0, am=0.0, blank=0, fastemit_lambda=0.0, scale=None):
    """reference()'s (costs [N], dF [N,T,V], dG [N,U,V]) in float64, from the factor formula and the chain rule.

    Per utterance, with Ef = exp(f - mf), Eg = exp(g - mg), S = Ef Eg^T, sg = rowsum Eg, A = Ef ug, the occupancies
    of the smoothed lattice Bk (blank) and Lb = (1 + lambda) e_y (label), both times scale[b], and O = Bk + Lb:
      full term (c):   dF = c (Ef * ((O/S) Eg) - sparse_f),      dG = c (Eg * ((O/S)^T Ef) - sparse_g)
      lm-only term:    dG += lml (O_u Eg / sg - sparse_g)           O_u = sum_t O
      am-only term:    dF += lma (O_t Ef ug / A - sparse_f)         O_t = sum_u O
      through ug:      h[v] = lma (sum_{b,t} O_t Ef[t,v] / A(t) - Z[v] / ug[v]),  dG += Eg / (M sg) (h - hbar_u)
    sparse_f / sparse_g put Bk on the blank column and Lb on the label columns; Z[v] sums them over the batch,
    hbar_u = sum_v Eg[u,v] h[v] / sg(u).  One utterance at a time, plus one batch vector for h."""
    N, T, V = trans.shape
    U = pred.shape[1]
    c = 1.0 - lm - am
    labels = np.asarray(labels)
    s = np.ones(N) if scale is None else np.asarray(scale, np.float64)
    ext = extents(act_lens, label_lens, T, U)
    preds = []   # (g, Eg, mg, sg) of the valid rows
    for b, (_, Ub) in enumerate(ext):
        g = np.asarray(pred[b, :Ub], np.float64)
        Eg, mg = _exp_rows(g)
        preds.append((g, Eg, mg, Eg.sum(axis=1)))
    M = sum(Ub for _, Ub in ext)
    if am != 0.0:
        ug = sum((Eg / sg[:, None]).sum(axis=0) for _, Eg, _, sg in preds) / M + FLT_MIN
        hsum, Z = np.zeros(V), np.zeros(V)
    costs, dF, dG = np.zeros(N), np.zeros((N, T, V)), np.zeros((N, U, V))
    for b, (Tb, Ub) in enumerate(ext):
        g, Eg, mg, sg = preds[b]
        f = np.asarray(trans[b, :Tb], np.float64)
        Ef, mf = _exp_rows(f)
        S = Ef @ Eg.T
        lse = mf[:, None] + mg[None, :] + np.log(S)
        Lg = mg + np.log(sg)
        if am != 0.0:
            A = Ef @ ug
            La = mf + np.log(A)
        y = labels[b, :Ub - 1].astype(np.int64) if Ub > 1 else np.zeros(0, np.int64)

        def lp(k):
            n = len(k)
            fk, gk = f[:, k], g[np.arange(n), k][None, :]
            out = np.zeros((Tb, n))
            if c != 0.0:
                out += c * (fk + gk - lse[:, :n])
            if lm != 0.0:
                out += lm * (gk - Lg[None, :n])
            if am != 0.0:
                out += am * (fk + np.log(ug[k])[None, :] - La[:, None])
            return out

        lpb, lpy = lp(np.full(Ub, blank, np.int64)), lp(y)
        alpha, beta, ll = lattice(lpb, lpy)
        costs[b] = -ll
        beta_next = np.full((Tb, Ub), -np.inf)   # beta(t+1, u), with the final blank into beta(T_b, U_b-1) = 0
        beta_next[:Tb - 1] = beta[1:]
        beta_next[Tb - 1, Ub - 1] = 0.0
        Bk = s[b] * np.exp(alpha + lpb + beta_next - ll)
        Lb = s[b] * (1.0 + fastemit_lambda) * np.exp(alpha[:, :Ub - 1] + lpy + beta[:, 1:] - ll)
        O = Bk.copy()
        O[:, :Ub - 1] += Lb
        sp_f, sp_g = np.zeros((Tb, V)), np.zeros((Ub, V))
        sp_f[:, blank] += Bk.sum(axis=1)
        sp_g[:, blank] += Bk.sum(axis=0)
        for u in range(Ub - 1):
            sp_f[:, y[u]] += Lb[:, u]
            sp_g[u, y[u]] += Lb[:, u].sum()
        dFb, dGb = -(c + am) * sp_f, -(c + lm) * sp_g
        if c != 0.0:
            W = O / S
            dFb += c * Ef * (W @ Eg)
            dGb += c * Eg * (W.T @ Ef)
        if lm != 0.0:
            dGb += lm * (O.sum(axis=0) / sg)[:, None] * Eg
        if am != 0.0:
            wt = O.sum(axis=1) / A   # O_t / A(t)
            dFb += am * wt[:, None] * Ef * ug[None, :]
            hsum += wt @ Ef
            Z[blank] += Bk.sum()
            np.add.at(Z, y, Lb.sum(axis=0))
        dF[b, :Tb], dG[b, :Ub] = dFb, dGb
    if am != 0.0:
        h = am * (hsum - Z / ug)
        for b, (_, Ub) in enumerate(ext):
            _, Eg, _, sg = preds[b]
            R = Eg / sg[:, None]
            dG[b, :Ub] += R * (h[None, :] - (R @ h)[:, None]) / M
    return costs, dF, dG
