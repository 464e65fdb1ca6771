"""fp64 CPU reference of the gradient options (FastEmit, clamp) for the tests.  Test infrastructure only.

Built on the unregularised oracle (oracle/rnnt_oracle.c through pyoracle): its dense gradient and, per
utterance, its alpha / beta lattices.  FastEmit(lambda) adds, per valid cell with a label,
    lambda * e_y * (p_k - [k = y_u]),   e_y = exp(alpha(t,u) + lp_y(t,u) + beta(t,u+1) - ll),
which turns the oracle's g_k = p_k (e_b + e_y) - [k = blank] e_b - [k = y_u] e_y into
    g_k = p_k (occ + lambda e_y) - [k = blank] e_b - [k = y_u] (1 + lambda) e_y.
ll is the oracle's backward log-likelihood beta(0,0), the value it normalises its own gradient with.
clamp > 0 clips the result element-wise.  Costs are the oracle's, whatever the options.
"""
import numpy as np

from oracle import pyoracle


def rnnt_logits_reg(acts, labels, act_lens, label_lens, blank=0, fastemit_lambda=0.0, clamp=-1.0):
    """(costs [N], dense float64 gradient w.r.t. the logits [N,T,U,V]) with the gradient options."""
    acts = np.ascontiguousarray(acts, dtype=np.float64)
    labels = np.asarray(labels, dtype=np.int32).reshape(acts.shape[0], -1)
    act_lens = np.asarray(act_lens, dtype=np.int32)
    label_lens = np.asarray(label_lens, dtype=np.int32)
    costs, grads, _ = pyoracle.rnnt_logits(acts, labels, act_lens, label_lens, blank)
    lam = float(fastemit_lambda)
    if lam > 0.0:
        for b in range(acts.shape[0]):
            T, U = int(act_lens[b]), int(label_lens[b]) + 1
            if U < 2:
                continue        # no label transitions: FastEmit leaves the utterance alone
            x = np.ascontiguousarray(acts[b:b + 1, :T, :U])
            y = np.ascontiguousarray(labels[b:b + 1, :U - 1])
            _, _, _, alpha, beta = pyoracle.rnnt_logits(x, y, [T], [U - 1], blank, want_lattice=True)
            lp = pyoracle.log_softmax_np(x[0, :, :U - 1])                            # [T, U-1, V]
            yy = y[0]
            lpy = np.take_along_axis(lp, np.broadcast_to(yy[None, :, None], (T, U - 1, 1)), axis=2)[..., 0]
            e_y = np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - beta[0, 0])         # [T, U-1]
            add = lam * e_y[..., None] * np.exp(lp)
            tt, uu = np.meshgrid(np.arange(T), np.arange(U - 1), indexing="ij")
            add[tt, uu, yy[uu]] -= lam * e_y
            grads[b, :T, :U - 1] += add
    if clamp > 0:
        grads = np.clip(grads, -clamp, clamp)
    return costs, grads
