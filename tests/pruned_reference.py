"""fp64 CPU reference of the pruned RNN-T loss and of its pruning ranges (DESIGN.md §8), for the tests.

pruned_loss(): logits [N, maxT, R, V], row (b, t, s) = lattice cell (t, ranges[b, t] + s).  The lattice is the
dense [T_b, U_b] one; a cell no row covers has log-zero blank and label factors; a covered cell takes the blank
log-prob and, for u < U_b - 1, the log-prob of y_u from its row.  Rows with t >= T_b, u < 0 or u >= U_b are
padding (zero gradient).  A valid row's gradient is the dense formula at (b, t, u), with the gradient options of
tests/regularized_reference.py.  No surviving path: cost +inf, zero gradient.

prune_ranges(): the window starts of include/rnnt.h (rnnt_b200_add_joint_prune_ranges) from the blank / label
occupancies of the simple (additive-joint) lattice, simple_occupancies().  Test infrastructure only.
"""
import numpy as np

NEG = -np.inf


def log_softmax(x):
    m = x.max(axis=-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(axis=-1, keepdims=True))


def lattice(lpb, lpy):
    """alpha, beta [T, U] and ll (natural log) of the lattice with blank log-probs lpb [T, U] and label
    log-probs lpy [T, U-1]; beta's virtual cell beta(T, U-1) = 0."""
    T, U = lpb.shape
    alpha = np.full((T, U), NEG)
    beta = np.full((T, U), NEG)
    alpha[0, 0] = 0.0
    for t in range(T):
        for u in range(U):
            if t == 0 and u == 0:
                continue
            a = alpha[t - 1, u] + lpb[t - 1, u] if t > 0 else NEG
            b = alpha[t, u - 1] + lpy[t, u - 1] if u > 0 else NEG
            alpha[t, u] = np.logaddexp(a, b)
    for t in range(T - 1, -1, -1):
        for u in range(U - 1, -1, -1):
            a = (beta[t + 1, u] if t < T - 1 else (0.0 if u == U - 1 else NEG)) + lpb[t, u]
            b = beta[t, u + 1] + lpy[t, u] if u < U - 1 else NEG
            beta[t, u] = np.logaddexp(a, b)
    return alpha, beta, beta[0, 0]


def pruned_factors(lp, labels_b, ranges_b, T, U, blank):
    """(lpb [T,U], lpy [T,U-1], cell [T,R] u of each row or -1 for padding) of one utterance; lp [maxT,R,V]."""
    R = lp.shape[1]
    lpb = np.full((T, U), NEG)
    lpy = np.full((T, max(U - 1, 0)), NEG)
    cell = np.full((lp.shape[0], R), -1, np.int64)
    for t in range(T):
        for s in range(R):
            u = int(ranges_b[t]) + s
            if 0 <= u < U:
                cell[t, s] = u
                lpb[t, u] = lp[t, s, blank]
                if u < U - 1:
                    lpy[t, u] = lp[t, s, labels_b[u]]
    return lpb, lpy, cell


def pruned_loss(logits, labels, act_lens, label_lens, ranges, blank=0, fastemit_lambda=0.0, clamp=-1.0):
    """(costs [N], gradient [N, maxT, R, V]) in float64."""
    logits = np.asarray(logits, dtype=np.float64)
    N, maxT, R, V = logits.shape
    labels = np.asarray(labels).reshape(N, -1)
    ranges = np.asarray(ranges, dtype=np.int64)
    costs = np.zeros(N)
    grads = np.zeros_like(logits)
    lam = float(fastemit_lambda)
    for b in range(N):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lp = log_softmax(logits[b])
        lpb, lpy, cell = pruned_factors(lp, labels[b], ranges[b], T, U, blank)
        alpha, beta, ll = lattice(lpb, lpy)
        if ll == NEG:
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
                g = p * (occ + lam * e_y)
                g[blank] -= e_b
                if u < U - 1:
                    g[labels[b, u]] -= (1.0 + lam) * e_y
                grads[b, t, s] = np.clip(g, -clamp, clamp) if clamp > 0 else g
    return costs, grads


def simple_occupancies(trans, pred, labels, act_lens, label_lens, blank=0):
    """Per utterance (e_b [T_b, U_b], e_y [T_b, U_b - 1]) of the additive joint logits trans[t] + pred[u]; e_b at
    t = T_b - 1 is not needed by the ranges and left zero."""
    trans, pred = np.asarray(trans, np.float64), np.asarray(pred, np.float64)
    out = []
    for b in range(trans.shape[0]):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lp = log_softmax(trans[b, :T, None, :] + pred[b, None, :U, :])   # [T, U, V]
        lpb = lp[:, :, blank]
        y = np.asarray(labels[b][:U - 1], np.int64)
        lpy = lp[:, np.arange(U - 1), y] if U > 1 else np.zeros((T, 0))
        alpha, beta, ll = lattice(lpb, lpy)
        e_b = np.zeros((T, U))
        e_b[:T - 1] = np.exp(alpha[:T - 1] + lpb[:T - 1] + beta[1:] - ll)
        e_y = np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - ll)
        out.append((e_b, e_y))
    return out


def window_scores(e_b, e_y, t, R):
    """k2's criterion for every start a in [0, E] of frame t."""
    U = e_b.shape[1]
    E = max(U - R, 0)
    return np.array([e_b[t, a:min(a + R, U)].sum() - (e_y[t, a - 1] if a > 0 else 0.0) for a in range(E + 1)])


def prune_ranges(occupancies, maxT, R):
    """[N, maxT] int32 window starts; also the smallest margin between a frame's best and runner-up score."""
    N = len(occupancies)
    ranges = np.zeros((N, maxT), np.int32)
    margin = np.inf
    for b, (e_b, e_y) in enumerate(occupancies):
        T, U = e_b.shape
        E = max(U - R, 0)
        s = np.full(maxT, E, np.int64)
        for t in range(1, T - 1):
            sc = window_scores(e_b, e_y, t, R)
            s[t] = int(np.argmax(sc))     # the first maximum: the smallest a
            if sc.size > 1:
                top = np.sort(sc)[-2:]
                margin = min(margin, top[1] - top[0])
        s[0] = 0
        if T > 1:
            s[T - 1] = E
        for t in range(T - 2, -1, -1):
            s[t] = min(max(s[t], s[t + 1] - (R - 1)), s[t + 1])
        ranges[b] = s
    return ranges, margin


def check_range_properties(ranges, act_lens, label_lens, R):
    """The structural properties of include/rnnt.h; raises AssertionError naming the first one broken."""
    for b in range(ranges.shape[0]):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        E = max(U - R, 0)
        s = np.asarray(ranges[b], np.int64)
        assert (s[T:] == E).all(), "frames past T_b start at E"
        s = s[:T]
        assert ((s >= 0) & (s <= E)).all(), "starts inside [0, E]"
        assert (np.diff(s) >= 0).all(), "non-decreasing"
        assert (np.diff(s) <= R - 1).all(), "consecutive windows overlap"
        assert s[T - 1] + R - 1 >= U - 1 or T == 1, "the last frame covers U_b - 1"
        # T_b > 1: s[0] == 0 leaves a path; without one (E > (T_b-1)(R-1)) s[0] > 0.  The sweep only raises s[0]
        # to s[1] - (R-1), so a frame-1 start beyond R-1 can lose a path that existed (DESIGN.md §8).  T_b == 1 keeps
        # s[0] = 0 whatever E is.
        if T > 1 and E > (T - 1) * (R - 1):
            assert s[0] > 0, "no path: s[0] > 0"


def random_monotone_ranges(rng, act_lens, label_lens, maxT, R):
    """Feasible non-decreasing windows: s[0] = 0, steps in [0, R-1], the last frame reaching U_b - 1 when it can."""
    N = len(act_lens)
    out = np.zeros((N, maxT), np.int32)
    for b in range(N):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        E = max(U - R, 0)
        s = np.zeros(maxT, np.int64)
        for t in range(1, T):
            need = E - s[t - 1]
            left = T - 1 - t          # steps still to come after this one
            lo = max(0, need - left * (R - 1))
            s[t] = s[t - 1] + min(R - 1, max(lo, int(rng.integers(0, R))))
        s[:T] = np.minimum(s[:T], E)
        s[T:] = E
        out[b] = s
    return out
