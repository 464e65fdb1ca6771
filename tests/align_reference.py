"""fp64 CPU reference of forced alignment (DESIGN.md §12, include/rnnt.h rnnt_b200_align), for the tests.

The factors are the loss's: pruned_reference.pruned_factors (dense: R = maxU, ranges == 0), natural-log blank
log-probs lpb [T, U] and label log-probs lpy [T, U-1], uncovered pruned cells at log zero.  No delay penalty.

    regular   a(0,0) = 0,  a(t,u) = max(a(t-1,u) + lpb(t-1,u), a(t,u-1) + lpy(t,u-1)),  best = a(T-1,U-1) + lpb(T-1,U-1)
    modified  a(0,0) = 0,  a(t,u) = max(a(t-1,u) + lpb(t-1,u), a(t-1,u-1) + lpy(t-1,u-1)),  best = a(T, U-1)

Tie rule: the label predecessor wins only when strictly greater, so equal partial paths emit labels early.
frames[j] is the frame of label j on the best path; no path (best = -inf): frames -1; a NaN factor: score NaN,
frames -1.  Test infrastructure only.
"""
import itertools

import numpy as np

import pruned_reference as pr

NEG = -np.inf


def align_factors(lpb, lpy, modified=False):
    """(score, frames [U-1] int) of one utterance's factors."""
    T, U = lpb.shape
    frames = np.full(U - 1, -1, np.int64)
    if np.isnan(lpb).any() or np.isnan(lpy).any():
        return np.nan, frames
    rows = T + 1 if modified else T
    a = np.full((rows, U), NEG)
    lab = np.zeros((rows, U), bool)   # the decision: label predecessor
    a[0, 0] = 0.0
    if modified:
        # row t depends on row t-1 only
        for t in range(1, rows):
            stay = a[t - 1] + lpb[t - 1]
            left = np.concatenate(([NEG], a[t - 1, :U - 1] + lpy[t - 1]))
            lab[t] = left > stay
            a[t] = np.where(lab[t], left, stay)
    else:
        # anti-diagonal n = t + u depends on diagonal n-1 only
        for n in range(1, T + U - 1):
            us = np.arange(max(0, n - T + 1), min(n, U - 1) + 1)
            ts = n - us
            tp, up = np.maximum(ts - 1, 0), np.maximum(us - 1, 0)
            stay = np.where(ts > 0, a[tp, us] + lpb[tp, us], NEG)
            left = np.where(us > 0, a[ts, up] + (lpy[ts, up] if U > 1 else NEG), NEG)
            lab[ts, us] = left > stay
            a[ts, us] = np.where(lab[ts, us], left, stay)
    best = a[T, U - 1] if modified else a[T - 1, U - 1] + lpb[T - 1, U - 1]
    if best == NEG:
        return NEG, frames
    t, u = (T, U - 1) if modified else (T - 1, U - 1)
    while t > 0 or u > 0:
        if lab[t, u]:
            frames[u - 1] = t - 1 if modified else t
            u -= 1
            if modified:
                t -= 1
        else:
            t -= 1
    return best, frames


def utterance_factors(logits_b, labels_b, ranges_b, T, U, blank):
    return pr.pruned_factors(pr.log_softmax(np.asarray(logits_b, np.float64)), labels_b, ranges_b, T, U, blank)[:2]


def align(logits, labels, act_lens, label_lens, ranges=None, blank=0, modified=False):
    """(scores [N], frames [N, maxU-1]) of logits [N, maxT, R, V]; ranges None: dense logits (R = maxU)."""
    logits = np.asarray(logits, np.float64)
    N, maxT, R, V = logits.shape
    labels = np.asarray(labels).reshape(N, -1)
    maxU = labels.shape[1] + 1
    ranges = np.zeros((N, maxT), np.int64) if ranges is None else np.asarray(ranges, np.int64)
    scores = np.zeros(N)
    frames = np.full((N, maxU - 1), -1, np.int64)
    for b in range(N):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lpb, lpy = utterance_factors(logits[b], labels[b], ranges[b], T, U, blank)
        scores[b], frames[b, :U - 1] = align_factors(lpb, lpy, modified)
    return scores, frames


def valid_alignment(frames_b, T, U, modified=False):
    """frames_b [U-1] (only the first U-1 entries are read) is an alignment of the topology."""
    f = np.asarray(frames_b[:U - 1], np.int64)
    if len(f) == 0:
        return True
    if f.min() < 0 or f.max() > T - 1:
        return False
    d = np.diff(f)
    return bool((d > 0).all() if modified else (d >= 0).all())


def rescore_factors(frames_b, lpb, lpy, modified=False):
    """fp64 log-probability of the alignment frames_b [U-1] (label j at frame frames_b[j])."""
    T, U = lpb.shape
    f = list(np.asarray(frames_b[:U - 1], np.int64))
    s, u = 0.0, 0
    for t in range(T):
        if modified:
            if u < U - 1 and f[u] == t:
                s += lpy[t, u]
                u += 1
            else:
                s += lpb[t, u]
        else:
            while u < U - 1 and f[u] == t:
                s += lpy[t, u]
                u += 1
            s += lpb[t, u]
    return s


def rescore(frames, logits, labels, act_lens, label_lens, ranges=None, blank=0, modified=False):
    """[N] fp64 log-probabilities of the alignments frames [N, maxU-1] under logits [N, maxT, R, V]."""
    logits = np.asarray(logits, np.float64)
    N, maxT = logits.shape[:2]
    labels = np.asarray(labels).reshape(N, -1)
    ranges = np.zeros((N, maxT), np.int64) if ranges is None else np.asarray(ranges, np.int64)
    out = np.zeros(N)
    for b in range(N):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lpb, lpy = utterance_factors(logits[b], labels[b], ranges[b], T, U, blank)
        out[b] = rescore_factors(frames[b], lpb, lpy, modified)
    return out


def all_alignments(T, U, modified=False):
    """Every alignment of a T x U lattice, as tuples of U-1 frames."""
    if modified:
        return list(itertools.combinations(range(T), U - 1))
    return list(itertools.combinations_with_replacement(range(T), U - 1))


def brute_force(lpb, lpy, modified=False):
    """(best score, its frames, log of the number of paths, logsumexp over all paths) by enumeration; -inf and
    None without a path."""
    T, U = lpb.shape
    paths = all_alignments(T, U, modified)
    if not paths:
        return NEG, None, NEG, NEG
    scores = np.array([rescore_factors(np.array(p), lpb, lpy, modified) for p in paths])
    k = int(np.argmax(scores))
    return scores[k], np.array(paths[k]), np.log(len(paths)), np.logaddexp.reduce(scores)


def random_alignment(rng, T, U, modified=False):
    """A uniformly drawn alignment (frames [U-1]), or None when the topology has none."""
    if modified:
        if U - 1 > T:
            return None
        return np.sort(rng.choice(T, U - 1, replace=False))
    return np.sort(rng.integers(0, T, U - 1))


def plant(rng, logits_b, labels_b, frames_b, T, U, blank=0, boost=10.0, ranges_b=None, modified=False):
    """Add `boost` to the logits of every transition of the alignment frames_b (in place): the blank of each frame
    and each label at its frame.  ranges_b: logits_b is pruned ([maxT, R, V], row s = cell ranges_b[t] + s)."""
    def row(t, u):
        return (t, u - int(ranges_b[t])) if ranges_b is not None else (t, u)
    u = 0
    for t in range(T):
        if modified:
            if u < U - 1 and frames_b[u] == t:
                logits_b[row(t, u) + (labels_b[u],)] += boost
                u += 1
            else:
                logits_b[row(t, u) + (blank,)] += boost
        else:
            while u < U - 1 and frames_b[u] == t:
                logits_b[row(t, u) + (labels_b[u],)] += boost
                u += 1
            logits_b[row(t, u) + (blank,)] += boost
