"""The fp64 pruned-loss reference (tests/pruned_reference.py) against the dense oracle and torch autograd, its
ranges against their structural properties, and the argument rules of the pruned C-ABI entries.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from pruned_reference import (check_range_properties, lattice, log_softmax, pruned_factors, pruned_loss,
                              prune_ranges, random_monotone_ranges, simple_occupancies)


def inputs(seed, N, T, U, V, R, blank=0):
    rng = np.random.default_rng(seed)
    logits = rng.standard_normal((N, T, R, V)) * 2
    labels = rng.choice(np.array([k for k in range(V) if k != blank]), size=(N, max(U - 1, 1))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return rng, logits, labels, tl, ul


@pytest.mark.parametrize("shape", [(3, 7, 5, 6), (2, 4, 1, 5), (2, 1, 4, 7), (3, 9, 6, 4)])
def test_identity_is_the_dense_loss(shape):
    """R = U, ranges == 0: the pruned loss is the RNN-T loss, costs and gradients."""
    N, T, U, V = shape
    _, logits, labels, tl, ul = inputs(1, N, T, U, V, U)
    c_ref, g_ref, _ = pyoracle.rnnt_logits(logits, labels[:, :U - 1], tl, ul, 0)
    c, g = pruned_loss(logits, labels[:, :U - 1], tl, ul, np.zeros((N, T), np.int32))
    assert np.allclose(c, c_ref, rtol=1e-12)
    assert np.allclose(g, g_ref, rtol=1e-10, atol=1e-13)


def autograd_loss(logits, labels, tl, ul, ranges, blank=0):
    """-ll of the pruned lattice by a torch fp64 log-sum-exp DP, and its gradient."""
    x = torch.tensor(logits, dtype=torch.float64, requires_grad=True)
    lp = torch.log_softmax(x, dim=-1)
    total = 0.0
    for b in range(x.shape[0]):
        T, U = int(tl[b]), int(ul[b]) + 1
        ninf = torch.tensor(-np.inf, dtype=torch.float64)
        lpb = [[ninf] * U for _ in range(T)]
        lpy = [[ninf] * U for _ in range(T)]
        for t in range(T):
            for s in range(x.shape[2]):
                u = int(ranges[b, t]) + s
                if 0 <= u < U:
                    lpb[t][u] = lp[b, t, s, blank]
                    if u < U - 1:
                        lpy[t][u] = lp[b, t, s, int(labels[b, u])]
        alpha = [[None] * U for _ in range(T)]
        for t in range(T):
            for u in range(U):
                terms = []
                if t == 0 and u == 0:
                    terms.append(torch.zeros((), dtype=torch.float64))
                if t > 0:
                    terms.append(alpha[t - 1][u] + lpb[t - 1][u])
                if u > 0:
                    terms.append(alpha[t][u - 1] + lpy[t][u - 1])
                terms = [x for x in terms if torch.isfinite(x)]   # all-dead cells: no NaN through logsumexp
                alpha[t][u] = torch.logsumexp(torch.stack(terms), 0) if terms else torch.tensor(-np.inf)
        total = total - (alpha[T - 1][U - 1] + lpb[T - 1][U - 1])
    total.backward()
    return x.grad.numpy()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gradient_is_autograd_of_the_pruned_lattice(seed):
    N, T, U, V, R = 3, 6, 5, 4, 3
    rng, logits, labels, tl, ul = inputs(seed, N, T, U, V, R)
    ranges = random_monotone_ranges(rng, tl, ul, T, R)
    if ranges[1, 1] <= R - 2:   # a window hanging off the lattice's left edge: its row at u = -1 is padding
        ranges[1, 0] = -1       # (short utterances, U_b < R, hang off the right edge)
    c, g = pruned_loss(logits, labels, tl, ul, ranges)
    assert np.isfinite(c).all()
    g_ag = autograd_loss(logits, labels, tl, ul, ranges)
    assert np.allclose(g, g_ag, rtol=1e-9, atol=1e-12)


def test_no_path_is_inf_with_zero_gradient():
    N, T, U, V, R = 2, 4, 6, 5, 2
    _, logits, labels, tl, ul = inputs(3, N, T, U, V, R)
    tl[:], ul[:] = T, U - 1
    ranges = np.zeros((N, T), np.int32)       # utterance 0: a window that never moves cannot reach U-1
    ranges[1] = [0, 1, 2, 4]                  # utterance 1: a skipped label
    c, g = pruned_loss(logits, labels, tl, ul, ranges)
    assert np.isinf(c).all() and (c > 0).all()
    assert not g.any()


@pytest.mark.parametrize("R", [2, 3, 5])
def test_ranges_properties(R):
    rng = np.random.default_rng(R)
    N, T, U, V = 6, 12, 9, 7
    trans = rng.standard_normal((N, T, V)) * 2
    pred = rng.standard_normal((N, U, V)) * 2
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(1, T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0], tl[1], ul[1] = T, U - 1, 2, U - 1   # utterance 1 has no path unless R is large
    occ = simple_occupancies(trans, pred, labels, tl, ul)
    ranges, _ = prune_ranges(occ, T, R)
    check_range_properties(ranges, tl, ul, R)
    for b in range(N):                                # T_b > 1: a window start of 0 always leaves a path
        if ranges[b, 0] == 0 and tl[b] > 1:
            T_b, U_b = int(tl[b]), int(ul[b]) + 1
            lp = log_softmax(np.zeros((T, R, V)))
            lpb, lpy, _ = pruned_factors(lp, labels[b], ranges[b], T_b, U_b, 0)
            assert np.isfinite(lattice(lpb, lpy)[2])


def test_occupancies_sum_to_frame_mass():
    """e_b summed over u is one per frame (every path leaves each frame t < T-1 by exactly one blank)."""
    rng = np.random.default_rng(5)
    N, T, U, V = 2, 6, 4, 5
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl, ul = np.array([T, T], np.int32), np.array([U - 1, U - 1], np.int32)
    for e_b, _ in simple_occupancies(trans, pred, labels, tl, ul):
        assert np.allclose(e_b[:T - 1].sum(axis=1), 1.0)


# ---- argument rules of the pruned C-ABI entries (host buffers: every call must stop before device access) -----
@pytest.fixture(scope="module")
def lib():
    import warprnnt_pytorch.warp_rnnt as wr
    h = C.CDLL(wr.lib_path())
    P, I = C.c_void_p, C.c_int
    h.rnnt_b200_pruned_workspace_size.argtypes = [I, I, I, I, C.c_size_t, C.POINTER(C.c_size_t)]
    h.rnnt_b200_pruned_loss_async_ex.argtypes = [I, I, P, P, P, I, P, P, P, I, I, P, C.c_double, wr.rnntGradOptions,
                                                 P, wr.rnntOptions]
    h.rnnt_b200_pruned_forward.argtypes = [I, P, P, I, P, P, P, I, I, P, I, P, wr.rnntOptions]
    h.rnnt_b200_pruned_backward_ex.argtypes = [I, P, P, P, I, P, P, P, I, I, P, C.c_double, wr.rnntGradOptions, P,
                                               wr.rnntOptions]
    h.rnnt_b200_add_joint_prune_ranges.argtypes = [P, P, I, I, P, P, wr.rnntOptions]
    return wr, h


def call(lib, name, loc=1, **kw):
    """One entry with host buffers and otherwise valid arguments (N=1, T=U=2, V=4, R=2), overridden by keyword."""
    wr, h = lib
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    opt = wr.rnntOptions(loc=loc, num_threads=0, stream=None, blank_label=0, maxT=kw.pop("maxT", 2),
                         maxU=kw.pop("maxU", 2), batch_first=True)
    a = dict(dtype=0, layout=0, acts=p, grads=p, ranges=p, R=2, labels=p, ylen=p, xlen=p, V=4, N=1, costs=p,
             svec=None, scale=1.0, gopt=wr.rnntGradOptions(0.0, 0.0), ws=p, prep=1)
    a.update(kw)
    if name == "loss":
        return h.rnnt_b200_pruned_loss_async_ex(a["dtype"], a["layout"], a["acts"], a["grads"], a["ranges"], a["R"],
                                                a["labels"], a["ylen"], a["xlen"], a["V"], a["N"], a["costs"],
                                                a["scale"], a["gopt"], a["ws"], opt)
    if name == "forward":
        return h.rnnt_b200_pruned_forward(a["dtype"], a["acts"], a["ranges"], a["R"], a["labels"], a["ylen"],
                                          a["xlen"], a["V"], a["N"], a["costs"], a["prep"], a["ws"], opt)
    if name == "backward":
        return h.rnnt_b200_pruned_backward_ex(a["dtype"], a["acts"], a["grads"], a["ranges"], a["R"], a["labels"],
                                              a["ylen"], a["xlen"], a["V"], a["N"], a["svec"], a["scale"], a["gopt"],
                                              a["ws"], opt)
    return h.rnnt_b200_add_joint_prune_ranges(a["ylen"], a["xlen"], a["N"], a["R"], a["ranges"], a["ws"], opt)


PRUNED = ["loss", "forward", "backward"]


@pytest.mark.parametrize("name", PRUNED)
def test_pruned_entries_accept_the_valid_call(lib, name):
    assert call(lib, name, loc=0) == 3     # reaches the location check: every other argument passed


@pytest.mark.parametrize("name", PRUNED)
@pytest.mark.parametrize("bad", [dict(ranges=None), dict(acts=None), dict(labels=None), dict(ws=None),
                                 dict(R=0), dict(R=-3), dict(V=0), dict(N=0), dict(maxT=0), dict(maxU=0),
                                 dict(dtype=4), dict(dtype=-1), dict(gopt="nan"), dict(R=1 << 30, maxT=4)],
                         ids=lambda d: "-".join("%s=%s" % kv for kv in d.items()))
def test_pruned_entries_reject(lib, name, bad):
    wr, _ = lib
    bad = dict(bad)
    if "gopt" in bad and name == "forward":
        pytest.skip("the forward takes no gradient options")
    if bad.get("gopt") == "nan":
        bad["gopt"] = wr.rnntGradOptions(float("nan"), 0.0)
    assert call(lib, name, loc=0, **bad) == 2


def test_pruned_rejects_the_time_major_layout(lib):
    assert call(lib, "loss", loc=0, layout=1) == 2
    assert call(lib, "loss", loc=0, layout=2) == 2
    assert call(lib, "backward", loc=0, grads=None) == 2
    assert call(lib, "forward", loc=0, costs=None) == 2


@pytest.mark.parametrize("dtype", [0, 1, 2, 3])
def test_pruned_accepts_every_storage_type(lib, dtype):
    for name in PRUNED:
        assert call(lib, name, loc=0, dtype=dtype) == 3


@pytest.mark.parametrize("bad", [dict(R=1), dict(R=0), dict(ranges=None), dict(ws=None), dict(ylen=None),
                                 dict(xlen=None), dict(N=0), dict(maxT=0), dict(maxU=0), dict(maxU=1025)],
                         ids=lambda d: "-".join("%s=%s" % kv for kv in d.items()))
def test_prune_ranges_entry_rejects(lib, bad):
    assert call(lib, "ranges", **bad) == 2
    assert call(lib, "ranges", loc=0, R=2) == 2        # a CPU location is not a device call either


def test_pruned_workspace_size(lib):
    wr, h = lib
    n = C.c_size_t(0)
    assert h.rnnt_b200_pruned_workspace_size(10, 5, 3, 4, 4, C.byref(n)) == 0 and n.value > 0
    dense = wr.workspace_size(10, 5, 4, 4)
    assert h.rnnt_b200_pruned_workspace_size(10, 5, 5, 4, 4, C.byref(n)) == 0 and n.value == dense
    for args in [(0, 5, 3, 4), (10, 0, 3, 4), (10, 5, 0, 4), (10, 5, 3, 0)]:
        assert h.rnnt_b200_pruned_workspace_size(*args, 4, C.byref(n)) == 2
    assert h.rnnt_b200_pruned_workspace_size(10, 5, 3, 4, 4, None) == 2
