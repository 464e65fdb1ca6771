"""fp64 reference and gradient tolerance for the additive joint (AddJointRNNTLoss).

The reference materialises h[b,t,u,v] = trans[b,t,v] + pred[b,u,v] in float64, runs the oracle on it and
reduces the logits gradient onto the two factors.

Tolerance of a factor gradient, per utterance, on its valid rows only (t < act_len for dF, u <= label_len
for dG; the padded rows must be exactly zero):
  * the blank column and the utterance's label columns carry the O(1) cancellation of the lattice terms
    against the dense term:  |g - g_ref| <= 1e-4 |g_ref| + 2e-6;
  * every other column is a pure dense term (Ef * P or Eg * Q, sums of positive products, no cancellation):
    |g - g_ref| <= 1e-4 |g_ref| + 1e-9.  At large V most of those elements are far below 2e-6, so the
    blank/label floor would hide a relative error of a whole vocabulary tile there.
"""
import numpy as np

from oracle import pyoracle

RTOL = 1e-4
FLOOR_SPARSE = 2e-6   # blank and label columns
FLOOR_DENSE = 1e-9    # every other column


def reference(trans, pred, labels, tl, ul, blank):
    """(costs [N], dF [N,T,V], dG [N,U,V]) in float64, one utterance at a time (bounded memory)."""
    N, T, V = trans.shape
    U = pred.shape[1]
    costs = np.zeros(N)
    dF = np.zeros((N, T, V))
    dG = np.zeros((N, U, V))
    for b in range(N):
        acts = trans[b:b + 1, :, None, :].astype(np.float64) + pred[b:b + 1, None, :, :].astype(np.float64)
        lab = labels[b:b + 1] if labels.size else np.zeros((1, 0), np.int32)
        c, g, _ = pyoracle.rnnt_logits(acts, lab, tl[b:b + 1], ul[b:b + 1], blank)
        costs[b] = c[0]
        dF[b] = g[0].sum(axis=1)
        dG[b] = g[0].sum(axis=0)
        del acts, g
    return costs, dF, dG


def sparse_columns(labels, ul, b, blank):
    """The blank and the labels of utterance b: the columns whose gradient has lattice terms."""
    cols = {int(blank)}
    if labels.size:
        cols.update(int(y) for y in labels[b, :int(ul[b])])
    return np.array(sorted(cols), dtype=np.int64)


def grad_mismatch(got, ref, rows, labels, ul, blank, what, batch=None, floor_sparse=FLOOR_SPARSE,
                  floor_dense=FLOOR_DENSE):
    """Problems of a factor gradient against the reference (empty list: within tolerance).

    got, ref: [N, R, V]; rows[b]: valid rows of utterance b.  `batch`: utterance indices of got/ref's
    first axis (default 0..N-1), for references computed on a subset of the batch.
    Each problem names the utterance and the floor the data would need (max of |g - g_ref| - 1e-4 |g_ref|)."""
    problems = []
    batch = range(got.shape[0]) if batch is None else batch
    for i, b in enumerate(batch):
        n = int(rows[b])
        pad = got[i, n:]
        if pad.size and np.any(pad != 0):
            problems.append("%s[%d]: padded rows not zero (max |g| %.3g)" % (what, b, np.abs(pad).max()))
        g, r = got[i, :n].astype(np.float64), ref[i, :n]
        if not n:
            continue
        sparse = np.zeros(g.shape[-1], bool)
        sparse[sparse_columns(labels, ul, b, blank)] = True
        excess = np.abs(g - r) - RTOL * np.abs(r)
        for mask, floor, kind in ((~sparse, floor_dense, "dense"), (sparse, floor_sparse, "blank/label")):
            if not mask.any():
                continue
            worst = float(excess[:, mask].max())
            if not worst <= floor:
                t, v = np.unravel_index(np.argmax(np.where(mask, excess, -np.inf)), excess.shape)
                problems.append("%s[%d] %s columns: needs floor %.3g > %.0e (row %d col %d: got %.9g ref %.9g)" % (
                    what, b, kind, worst, floor, t, v, g[t, v], r[t, v]))
    return problems


def assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, batch=None, scale=None,
                       floor_sparse=FLOOR_SPARSE, floor_dense=FLOOR_DENSE):
    """Costs to rtol 1e-5; dF and dG to the column-wise tolerance above (floors overridable where a shape
    needs more, with the measured number beside the override).  `scale[b]`: the upstream gradient of
    utterance b (the reference is scaled by it)."""
    batch = list(range(len(c_ref))) if batch is None else list(batch)
    assert np.allclose(costs, c_ref, rtol=1e-5, atol=1e-5), np.abs(costs - c_ref).max()
    s = np.ones(len(batch)) if scale is None else np.asarray(scale, np.float64)
    rows_g = np.asarray(ul) + 1
    floors = dict(floor_sparse=floor_sparse, floor_dense=floor_dense)
    problems = grad_mismatch(dF, dF_ref * s[:, None, None], tl, labels, ul, blank, "dF", batch, **floors) + \
        grad_mismatch(dG, dG_ref * s[:, None, None], rows_g, labels, ul, blank, "dG", batch, **floors)
    assert not problems, "\n".join(problems)
