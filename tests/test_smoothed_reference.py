"""The fp64 reference of the smoothed additive joint (tests/smoothed_reference.py) against its defining properties,
and the argument rules of the smoothed C-ABI entries.  No GPU."""
import ctypes as C
import math

import numpy as np
import pytest

import smoothed_reference as sr
from pruned_reference import lattice, log_softmax

SCALES = [(0.25, 0.0), (0.0, 0.25), (0.25, 0.1), (0.5, 0.5), (1.0, 0.0), (0.0, 1.0)]


def problem(seed=0, N=3, T=5, U=4, V=7, ragged=True):
    rng = np.random.default_rng(seed)
    trans = rng.standard_normal((N, T, V))
    pred = rng.standard_normal((N, U, V))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = np.array([T, T - 2, 3][:N] if ragged else [T] * N, np.int32)
    ul = np.array([U - 1, 1, U - 2][:N] if ragged else [U - 1] * N, np.int32)
    return trans, pred, labels, tl, ul


def test_zero_scales_equal_the_plain_joint():
    from joint_reference import reference
    trans, pred, labels, tl, ul = problem()
    c_ref, dF_ref, dG_ref = reference(trans.astype(np.float32), pred.astype(np.float32), labels, tl, ul, 0)
    f32 = lambda x: x.astype(np.float32).astype(np.float64)   # noqa: E731  the oracle saw float32 inputs
    c, dF, dG = sr.reference(f32(trans), f32(pred), labels, tl, ul)
    assert np.allclose(c, c_ref, rtol=1e-10)
    assert np.allclose(dF, dF_ref, atol=1e-10) and np.allclose(dG, dG_ref, atol=1e-10)


def test_lm_only_ignores_trans():
    trans, pred, labels, tl, ul = problem(1)
    c, dF, _ = sr.reference(trans, pred, labels, tl, ul, lm=1.0)
    assert not dF.any()
    direct = []
    for b in range(len(tl)):
        T, U = int(tl[b]), int(ul[b]) + 1
        lp = log_softmax(pred[b, :U])                                  # [U, V], the same for every frame
        lpb = np.repeat(lp[None, :, 0], T, axis=0)
        lpy = np.repeat(lp[None, np.arange(U - 1), labels[b, :U - 1]], T, axis=0)
        direct.append(-lattice(lpb, lpy)[2])
    assert np.allclose(c, direct, rtol=1e-12)
    assert np.allclose(sr.costs(trans + 3.0 * np.random.default_rng(5).standard_normal(trans.shape), pred, labels,
                                tl, ul, lm=1.0), c, rtol=1e-12)


@pytest.mark.parametrize("lm,am", SCALES)
def test_costs_invariant_to_row_shifts(lm, am):
    trans, pred, labels, tl, ul = problem(2)
    c = sr.costs(trans, pred, labels, tl, ul, lm, am)
    t2, p2 = trans.copy(), pred.copy()
    t2[0, 1] += 7.5
    t2[2, 0] -= 3.0
    p2[1, 0] += 11.0
    p2[0, 2] -= 4.0
    assert np.allclose(sr.costs(t2, p2, labels, tl, ul, lm, am), c, rtol=1e-10)


@pytest.mark.parametrize("lm,am", SCALES)
def test_torch_gradient_matches_central_differences(lm, am):
    trans, pred, labels, tl, ul = problem(3, N=2, T=3, U=3, V=5)
    scale = np.array([1.0, 0.5])
    _, dF, dG = sr.reference(trans, pred, labels, tl, ul, lm, am, scale=scale)
    eps = 1e-6

    def J(t, p):
        return float((sr.costs(t, p, labels, tl, ul, lm, am) * scale).sum())

    for x, d in ((trans, dF), (pred, dG)):
        num = np.zeros_like(x)
        for i in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[i] += eps
            xm[i] -= eps
            num[i] = (J(*((xp, pred) if x is trans else (trans, xp))) -
                      J(*((xm, pred) if x is trans else (trans, xm)))) / (2 * eps)
        assert np.allclose(d, num, atol=1e-7), np.abs(d - num).max()


def test_unigram_couples_the_batch():
    trans, pred, labels, tl, ul = problem(4)
    _, _, dG = sr.reference(trans, pred, labels, tl, ul, 0.1, 0.3, scale=[1.0, 0.0, 0.0])
    assert np.abs(dG[1, :int(ul[1]) + 1]).max() > 1e-6      # utterance 0's cost moves utterance 1's pred rows
    _, _, dG = sr.reference(trans, pred, labels, tl, ul, 0.3, 0.0, scale=[1.0, 0.0, 0.0])
    assert not dG[1:].any()                                # without the am-only term it does not


@pytest.mark.parametrize("lm,am", SCALES)
def test_padded_pred_rows_are_not_read(lm, am):
    trans, pred, labels, tl, ul = problem(5)
    c, dF, dG = sr.reference(trans, pred, labels, tl, ul, lm, am)
    p2 = pred.copy()
    for b in range(len(ul)):
        p2[b, int(ul[b]) + 1:] = 1e3 * np.random.default_rng(b).standard_normal(p2[b, int(ul[b]) + 1:].shape)
    c2, dF2, dG2 = sr.reference(trans, p2, labels, tl, ul, lm, am)
    assert np.array_equal(c, c2) and np.array_equal(dF, dF2) and np.array_equal(dG, dG2)
    for b in range(len(ul)):
        assert not dG[b, int(ul[b]) + 1:].any() and not dF[b, int(tl[b]):].any()


def assert_rel_close(got, want, rtol=1e-10):
    """Elementwise within rtol of the array's largest magnitude (the gradients hold exact zeros and tiny values)."""
    for g, w in zip(got, want):
        assert g.shape == w.shape
        assert np.abs(g - w).max() <= rtol * max(np.abs(w).max(), 1e-300), np.abs(g - w).max() / np.abs(w).max()


def assert_closed_form_matches(x, lm, am, **kw):
    trans, pred, labels, tl, ul = x
    got = sr.closed_form(trans, pred, labels, tl, ul, lm, am, **kw)
    want = sr.reference(trans, pred, labels, tl, ul, lm, am, **kw)
    assert_rel_close(got, want)
    return got


@pytest.mark.parametrize("lm,am", SCALES + [(0.0, 0.0), (0.6, 0.4)])   # c = 0 at (1, 0), (0, 1) and (0.6, 0.4)
def test_closed_form_equals_autograd(lm, am):
    got = assert_closed_form_matches(problem(20, N=3, T=6, U=5, V=9), lm, am)
    if lm == 1.0:
        assert not got[1].any()


@pytest.mark.parametrize("lm,am", [(0.25, 0.0), (0.25, 0.1), (0.0, 1.0)])
def test_closed_form_fastemit_and_signed_scale(lm, am):
    x = problem(21, N=3, T=5, U=4, V=8)
    assert_closed_form_matches(x, lm, am, fastemit_lambda=0.3, scale=np.array([0.5, -1.25, 2.0]))


@pytest.mark.parametrize("lm,am", [(0.25, 0.1), (0.5, 0.5)])
def test_closed_form_edges(lm, am):
    # one frame per utterance; blank = V - 1
    trans, pred, labels, _, ul = problem(22, N=3, T=4, U=4, V=6)
    labels = np.minimum(labels, 4).astype(np.int32)   # labels in 1..4, never the blank 5
    assert_closed_form_matches((trans, pred, labels, np.ones(3, np.int32), ul), lm, am, blank=5)
    # every U_b = 1: no labels, ug over N pred rows
    trans, pred, labels, tl, _ = problem(23, N=3, T=5, U=3, V=7)
    assert_closed_form_matches((trans, pred, labels, tl, np.zeros(3, np.int32)), lm, am)


@pytest.mark.parametrize("lm,am", [(0.25, 0.1), (0.0, 0.25), (0.0, 0.0)])
def test_closed_form_masked_vocabulary_columns(lm, am):
    trans, pred, labels, tl, ul = problem(24, N=3, T=5, U=4, V=10)
    labels = np.where(labels >= 7, labels - 6, labels).astype(np.int32)   # columns 7..9 are neither blank nor label
    trans[:, :, 7:] = -np.inf
    c, dF, dG = assert_closed_form_matches((trans, pred, labels, tl, ul), lm, am)
    assert np.all(np.isfinite(c)) and not dF[:, :, 7:].any()


def test_closed_form_zero_scales_equal_the_joint_reference():
    from joint_reference import reference
    trans, pred, labels, tl, ul = problem(25, N=3, T=6, U=5, V=8)
    f32 = lambda x: x.astype(np.float32).astype(np.float64)   # noqa: E731  the oracle saw float32 inputs
    c_ref, dF_ref, dG_ref = reference(trans.astype(np.float32), pred.astype(np.float32), labels, tl, ul, 0)
    assert_rel_close(sr.closed_form(f32(trans), f32(pred), labels, tl, ul), (c_ref, dF_ref, dG_ref))


def test_closed_form_reaches_the_training_shape_in_bounded_memory():
    """One C3-sized utterance (T 150, U 21, V 5000): the closed form holds O((T + U) V) per utterance."""
    rng = np.random.default_rng(26)
    N, T, U, V = 2, 150, 21, 5000
    trans = rng.standard_normal((N, T, V)).astype(np.float32)
    pred = rng.standard_normal((N, U, V)).astype(np.float32)
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl, ul = np.array([T, 97], np.int32), np.array([U - 1, 13], np.int32)
    c, dF, dG = sr.closed_form(trans, pred, labels, tl, ul, 0.25, 0.1)
    assert np.all(np.isfinite(c)) and np.isfinite(dF).all() and np.isfinite(dG).all()
    assert np.allclose(c, sr.costs(trans, pred, labels, tl, ul, 0.25, 0.1), rtol=1e-12)
    # every logit's gradient sums to 0 over v, and the am-only / lm-only / full terms each do: so do dF and dG rows
    assert np.abs(dF.sum(-1)).max() < 1e-9 and np.abs(dG.sum(-1)).max() < 1e-9


# ---- argument rules of the smoothed entries (host buffers, rejected before any device access) ----------------------
@pytest.fixture(scope="module")
def abi():
    import warprnnt_pytorch.warp_rnnt as wr
    from warprnnt_pytorch.joint import rnntSmoothOptions
    lib = C.CDLL(wr.lib_path())
    P = C.c_void_p
    fwd = lib.rnnt_b200_add_joint_smoothed_forward
    fwd.restype = C.c_int
    fwd.argtypes = [P, P, P, P, P, C.c_int, C.c_int, P, C.c_int, rnntSmoothOptions, P, wr.rnntOptions]
    bwd = lib.rnnt_b200_add_joint_smoothed_backward
    bwd.restype = C.c_int
    bwd.argtypes = [P, P, P, P, P, P, P, C.c_int, C.c_int, P, C.c_float, wr.rnntGradOptions, rnntSmoothOptions, P,
                    wr.rnntOptions]
    ws = lib.rnnt_b200_add_joint_smoothed_workspace_size
    ws.restype = C.c_int
    ws.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]
    return wr, rnntSmoothOptions, fwd, bwd, ws, lib


class Smoothed:
    """One smoothed entry with host buffers and otherwise valid arguments, overridden by keyword."""
    FWD = "f g labels ylen xlen V N costs prep smooth ws opt"
    BWD = "f g dF dG labels ylen xlen V N svec scale gopt smooth ws opt"

    def __init__(self, abi, which):
        self.wr, self.S, fwd, bwd, _, _ = abi
        self.fn = fwd if which == "forward" else bwd
        self.params = (self.FWD if which == "forward" else self.BWD).split()
        self.buf = (C.c_double * 64)()
        self.ibuf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1)

    def __call__(self, loc=1, maxT=2, maxU=2, blank=0, lm=0.25, am=0.1, **kw):
        opt = self.wr.rnntOptions(loc=loc, num_threads=0, stream=None, blank_label=blank, maxT=maxT, maxU=maxU,
                                  batch_first=True)
        args = dict(V=4, N=1, prep=1, scale=1.0, gopt=self.wr.rnntGradOptions(0.0, 0.0), smooth=self.S(lm, am), opt=opt)
        for q in self.params:
            if q not in args:
                args[q] = C.addressof(self.ibuf if q in ("labels", "ylen", "xlen") else self.buf)
        assert set(kw) <= set(self.params), kw
        args.update(kw)
        return self.fn(*[args[q] for q in self.params])


@pytest.fixture(params=["forward", "backward"])
def entry(request, abi):
    return Smoothed(abi, request.param)


BAD_SCALES = [(math.nan, 0.0), (0.0, math.nan), (math.inf, 0.0), (0.0, -math.inf), (-0.1, 0.0), (0.0, -1e-30),
              (0.6, 0.5), (1.0, 1e-6), (2.0, -1.0)]


def test_valid_calls_reach_the_location_check(entry):
    for lm, am in SCALES + [(0.0, 0.0), (0.6, 0.4), (0.3, 0.7), (0.1, 0.9)]:   # float32 sums up to 1 + 3e-8
        assert entry(loc=0, lm=lm, am=am) == 3, (lm, am)     # accepted: RNNT_CPU has no path


def test_bad_scales(entry):
    for lm, am in BAD_SCALES:
        assert entry(lm=lm, am=am) == 2, (lm, am)
        assert entry(loc=0, lm=lm, am=am) == 2, (lm, am)     # before the location


def test_null_pointers_and_extents(entry):
    optional = {"svec"}
    for q in entry.params:
        if q not in ("V", "N", "prep", "scale", "gopt", "smooth", "opt") and q not in optional:
            assert entry(**{q: None}) == 2, q
    for kw in ({"V": 0}, {"N": -1}, {"maxT": 0}, {"maxU": -2}, {"maxU": 1025}, {"blank": 4}):
        assert entry(**kw) == 2, kw
    assert entry(maxT=1 << 16, maxU=2, V=1 << 15) == 2      # the joint's 32-bit factor offsets
    assert entry(N=2, maxT=1 << 20, maxU=1024) == 2


def test_backward_rejects_a_clamp(abi):
    e = Smoothed(abi, "backward")
    assert e(loc=0, gopt=e.wr.rnntGradOptions(0.0, 1.0)) == 2
    assert e(loc=0, gopt=e.wr.rnntGradOptions(0.5, 0.0)) == 3


def test_workspace_size(abi):
    _, _, _, _, ws, lib = abi
    n, m = C.c_size_t(0), C.c_size_t(0)
    assert ws(7, 5, 3, 11, C.byref(n)) == 0
    lib.rnnt_b200_add_joint_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]
    assert lib.rnnt_b200_add_joint_workspace_size(7, 5, 3, 11, C.byref(m)) == 0
    assert n.value > m.value
    for args in ((0, 5, 3, 11), (7, 0, 3, 11), (7, 5, 0, 11), (7, 5, 3, 0)):
        assert ws(*args, C.byref(n)) == 2
    assert ws(7, 5, 3, 11, None) == 2


def test_python_scale_rules():
    from warprnnt_pytorch import joint
    assert joint.smooth_options(0.0, 0.0) is None
    assert joint.smooth_options(0.25, 0.0).lm_only_scale == 0.25
    assert joint.smooth_options(0.6, 0.4).am_only_scale == np.float32(0.4)   # sums to 1 as given
    for lm, am in BAD_SCALES:
        with pytest.raises(ValueError):
            joint.smooth_options(lm, am)
        with pytest.raises(ValueError):
            joint.AddJointRNNTLoss(lm_only_scale=lm, am_only_scale=am)
