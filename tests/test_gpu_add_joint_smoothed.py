"""Smoothed additive joint (lm_only_scale / am_only_scale, DESIGN.md §9) on the GPU against the fp64 reference
(tests/smoothed_reference.py), and its identity with the plain joint at scales (0, 0)."""
import numpy as np
import pytest
import torch

import smoothed_reference as sr
from joint_reference import assert_joint_close
from pruned_reference import prune_ranges

pytestmark = pytest.mark.gpu

SCALES = [(0.25, 0.0), (0.0, 0.25), (0.25, 0.1), (0.5, 0.5), (1.0, 0.0), (0.0, 1.0)]
# (N, T, U, V, blank): the dispatch each shape reaches
SHAPES = {
    "fused_V4k": (3, 40, 9, 1024, 0),          # grad_fused_kernel, A_MODE 3; joint_prep_row_kernel
    "fused_V_odd": (3, 37, 6, 131, 2),         # grad_fused_kernel, A_MODE 0; the warp prep kernel
    "two_kernel_U40": (2, 20, 40, 260, 0),     # U > 32: gemm_kernel dF / dG, MODE 3 operands
    "two_kernel_U40_V_odd": (2, 12, 40, 67, 1),   # MODE 0 operands, V % 4 != 0
    # the batch-wide column sums in their full 128-chunk form (rows >= 32 * 128, not a multiple of 128):
    "many_frames": (33, 125, 3, 40, 0),        # h over N*T = 4125 rows of Ef
    "many_labels": (65, 2, 65, 40, 1),         # ug over N*U = 4225 rows of Eg; dG in the 128-column tile (U > 64)
    "two_kernel_T70": (2, 70, 34, 67, 0),      # T > 64: dF in the 128-column tile with RNNT_B200_DF_TILE=128
}


def make_inputs(seed, N, T, U, V, blank, garbage=True):
    rng = np.random.default_rng(seed)
    trans = (rng.standard_normal((N, T, V)) * 2.0).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * 2.0).astype(np.float32)
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 0))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    if garbage:   # padded pred rows hold large values: they must not be read
        for b in range(N):
            pred[b, ul[b] + 1:] = rng.standard_normal(pred[b, ul[b] + 1:].shape) * 50.0
    return trans, pred, labels, tl, ul


def cuda(*xs):
    return [torch.as_tensor(x).cuda() for x in xs]


def run(trans, pred, labels, tl, ul, blank, lm=0.0, am=0.0, weights=None, reduction='none', **kw):
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = add_joint_rnnt_loss(tt, pp, lab, tl_, ul_, blank, reduction, lm_only_scale=lm, am_only_scale=am, **kw)
    w = torch.ones_like(out) if weights is None else torch.as_tensor(weights, dtype=torch.float32).cuda()
    (out * w).sum().backward()
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy()


@pytest.mark.parametrize("shape", list(SHAPES) + ["headline"])
def test_zero_scales_are_the_plain_joint_bitwise(shape):
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    from warprnnt_pytorch.joint import rnntSmoothOptions, joint_forward_call
    N, T, U, V, blank = SHAPES.get(shape, (128, 150, 21, 5000, 0))
    trans, pred, labels, tl, ul = make_inputs(7, N, T, U, V, blank)
    plain = run(trans, pred, labels, tl, ul, blank)
    smooth = run(trans, pred, labels, tl, ul, blank, 0.0, 0.0)
    for a, b in zip(plain, smooth):
        assert np.array_equal(a, b)
    # the smoothed entry itself with zero scales, on its own (larger) workspace
    tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
    c0, c1 = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
    joint_forward_call(tt, pp, lab, tl_, ul_, c0, True, blank, None)
    joint_forward_call(tt, pp, lab, tl_, ul_, c1, True, blank, rnntSmoothOptions(0.0, 0.0))
    assert torch.equal(c0, c1)
    if U > 2:
        _, r0 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, blank)
        _, r1 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, blank, lm_only_scale=0.0, am_only_scale=0.0)
        assert torch.equal(r0, r1)


# Floor override for am_only_scale > 0.  Every dG column then carries Eg / (M sg) (h[v] - hbar_u), a small difference
# of two large batch sums of lattice occupancies (DESIGN.md §9): the fp32 lattice's relative error there is what
# the blank / label columns see, so the dense 1e-9 floor is too tight.  Measured on an H100 80GB HBM3 at a 400 W
# power limit, the dG dense columns of this file need at most 3.15e-8 (two_kernel_U40, scales (0, 0.25)); dF and
# the plain floors hold everywhere.
FLOOR_DENSE_AM = 1e-7


def floors(am):
    return {"floor_dense": FLOOR_DENSE_AM} if am > 0 else {}


@pytest.mark.parametrize("lm,am", SCALES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_against_reference(shape, lm, am):
    N, T, U, V, blank = SHAPES[shape]
    trans, pred, labels, tl, ul = make_inputs(11, N, T, U, V, blank)
    w = np.linspace(0.5, 1.5, N)
    costs, dF, dG = run(trans, pred, labels, tl, ul, blank, lm, am, w)
    c_ref, dF_ref, dG_ref = sr.reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul, lm, am,
                                         blank, scale=w)
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, **floors(am))


@pytest.mark.parametrize("lm,am", [(0.25, 0.0), (0.25, 0.1)])
def test_fastemit_with_smoothing(lm, am):
    N, T, U, V, blank = SHAPES["fused_V4k"]
    trans, pred, labels, tl, ul = make_inputs(12, N, T, U, V, blank)
    costs, dF, dG = run(trans, pred, labels, tl, ul, blank, lm, am, fastemit_lambda=0.3)
    c_ref, dF_ref, dG_ref = sr.reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul, lm, am,
                                         blank, fastemit_lambda=0.3)
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, **floors(am))


@pytest.mark.parametrize("shape", ["fused_V4k", "two_kernel_U40"])
def test_two_calls_are_bitwise_identical(shape):
    N, T, U, V, blank = SHAPES[shape]
    trans, pred, labels, tl, ul = make_inputs(13, N, T, U, V, blank)
    a = run(trans, pred, labels, tl, ul, blank, 0.25, 0.1)
    b = run(trans, pred, labels, tl, ul, blank, 0.25, 0.1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


# The tuning hooks' smoothed paths run in test_gpu_tuning_hooks.py (the "smoothed" suite of hook_cases.py).


@pytest.mark.parametrize("lm,am", [(0.25, 0.0), (0.25, 0.1)])
def test_smoothed_ranges_equal_the_reference_windows(lm, am):
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    N, T, U, V, blank, R = 4, 30, 9, 64, 0, 3
    for seed in range(15, 65):   # the first seed whose best windows win by a margin fp32 cannot blur
        trans, pred, labels, tl, ul = make_inputs(seed, N, T, U, V, blank)
        occ = sr.smoothed_occupancies(trans, pred, labels, tl, ul, lm, am, blank)
        want, margin = prune_ranges(occ, T, R)
        if margin > 1e-4:
            break
    assert margin > 1e-4, "no seed with unambiguous windows"
    tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
    _, ranges = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, R, blank, lm_only_scale=lm, am_only_scale=am)
    assert np.array_equal(ranges.cpu().numpy(), want)


def test_icefall_style_step_against_fp64_torch():
    """Smoothed simple loss (lm 0.25, am 0.1) with its ranges, plus the pruned loss of a tanh joiner."""
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges, prune_joint_inputs, pruned_rnnt_loss
    from test_gpu_pruned import Model, torch_pruned
    N, T, U, D, V, R, blank, lm, am = 3, 7, 5, 6, 9, 3, 0, 0.25, 0.1
    rng = np.random.default_rng(52)
    labels_np = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl_np = np.array([T, T - 2, T - 1], np.int32)
    ul_np = np.array([U - 1, U - 3, U - 2], np.int32)
    enc_np, dec_np = rng.standard_normal((N, T, D)), rng.standard_normal((N, U, D))
    m32 = Model(D, V, 0).cuda()
    m64 = Model(D, V, 0).double()
    labels, tl, ul = cuda(labels_np, tl_np, ul_np)
    enc = torch.tensor(enc_np, dtype=torch.float32, device="cuda", requires_grad=True)
    dec = torch.tensor(dec_np, dtype=torch.float32, device="cuda", requires_grad=True)
    simple, ranges = add_joint_rnnt_loss_with_ranges(enc @ m32.am, dec @ m32.lm, labels, tl, ul, R, blank,
                                                     reduction='sum', lm_only_scale=lm, am_only_scale=am)
    enc_p, dec_p = prune_joint_inputs(enc, dec, ranges, R)
    pruned = pruned_rnnt_loss(torch.tanh(enc_p + dec_p) @ m32.out, labels, tl, ul, ranges, blank, reduction='sum')
    (0.5 * simple + pruned).backward()

    r = ranges.cpu().numpy()
    e64 = torch.tensor(enc_np, requires_grad=True)
    d64 = torch.tensor(dec_np, requires_grad=True)
    s64 = sr.torch_costs(e64 @ m64.am, d64 @ m64.lm, labels_np, tl_np, ul_np, lm, am, blank).sum()
    idx = torch.as_tensor(np.clip(r[:, :, None] + np.arange(R), 0, U - 1))
    dg = torch.gather(d64[:, None].expand(N, T, U, D), 2, idx[..., None].expand(N, T, R, D))
    p64 = torch_pruned(torch.tanh(e64[:, :, None] + dg) @ m64.out, labels_np, tl_np, ul_np, r, blank).sum()
    (0.5 * s64 + p64).backward()
    assert np.isclose(simple.item(), s64.item(), rtol=1e-5) and np.isclose(pruned.item(), p64.item(), rtol=1e-5)
    for a, b in ((enc.grad, e64.grad), (dec.grad, d64.grad), (m32.am.grad, m64.am.grad),
                 (m32.lm.grad, m64.lm.grad), (m32.out.grad, m64.out.grad)):
        a = a.double().cpu()
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (a - b).abs().max()


def test_reductions_grad_output_and_stream():
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N, T, U, V, blank = SHAPES["fused_V_odd"]
    trans, pred, labels, tl, ul = make_inputs(16, N, T, U, V, blank)
    lm, am = 0.25, 0.1
    c_none, dF, dG = run(trans, pred, labels, tl, ul, blank, lm, am)
    for red, k in (("sum", 1.0), ("mean", 1.0 / N)):
        c, dF2, dG2 = run(trans, pred, labels, tl, ul, blank, lm, am, reduction=red)
        assert np.allclose(c, c_none.sum() * k, rtol=1e-6)
        assert np.allclose(dF2, dF * k, rtol=1e-5, atol=1e-8) and np.allclose(dG2, dG * k, rtol=1e-5, atol=1e-8)
    g = np.array([0.5, -1.0, 2.0][:N])
    _, dF3, dG3 = run(trans, pred, labels, tl, ul, blank, lm, am, weights=g)
    c_ref, dF_ref, dG_ref = sr.reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul, lm, am,
                                         blank, scale=g)
    assert_joint_close(c_none, dF3, dG3, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, **floors(am))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        tt = torch.tensor(trans, device="cuda", requires_grad=True)
        pp = torch.tensor(pred, device="cuda", requires_grad=True)
        lab, tl_, ul_ = cuda(labels, tl, ul)
        out = AddJointRNNTLoss(blank, 'none', lm_only_scale=lm, am_only_scale=am)(tt, pp, lab, tl_, ul_)
        out.sum().backward()
    s.synchronize()
    assert np.array_equal(out.detach().cpu().numpy(), c_none)
    assert np.array_equal(tt.grad.cpu().numpy(), dF) and np.array_equal(pp.grad.cpu().numpy(), dG)


def test_value_errors():
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    from warprnnt_pytorch.joint import AddJointRNNTLoss, add_joint_rnnt_loss
    x = [torch.as_tensor(a).cuda() for a in make_inputs(17, 2, 4, 3, 8, 0)]
    for lm, am in ((float("nan"), 0.0), (-0.5, 0.0), (0.7, 0.4), (0.0, float("inf"))):
        with pytest.raises(ValueError):
            add_joint_rnnt_loss(*x, lm_only_scale=lm, am_only_scale=am)
        with pytest.raises(ValueError):
            add_joint_rnnt_loss_with_ranges(*x, 2, lm_only_scale=lm, am_only_scale=am)
        with pytest.raises(ValueError):
            AddJointRNNTLoss(lm_only_scale=lm, am_only_scale=am)
    with pytest.raises(ValueError):
        add_joint_rnnt_loss(*x, lm_only_scale=0.25, clamp=1.0)
