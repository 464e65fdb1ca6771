"""Smoothed additive joint (lm_only_scale / am_only_scale, DESIGN.md §9) at the boundaries of every kernel it runs,
against the closed-form fp64 reference (tests/smoothed_reference.py closed_form), at the training shapes, and with
non-finite values in the padding.

    plain-joint boundaries   every shape of test_gpu_add_joint_geometry: S tiles and split-K slabs (EpiStats<true>),
                             the fused gradient's chunks and the two-kernel gradient's tiles (SMOOTH epilogues)
    batch sums               joint_colsum_kernel's row chunks (smooth_chunks), the 256-column CTAs of the colsum,
                             unigram and h kernels, joint_unigram_grad_kernel's 256-item tiles, the warp loops of
                             joint_smooth_rows_kernel and joint_smooth_g_kernel
"""
import numpy as np
import pytest
import torch

import smoothed_reference as sr
import test_gpu_add_joint_geometry as geo
from joint_reference import FLOOR_DENSE, FLOOR_SPARSE, assert_joint_close
from test_gpu_add_joint_smoothed import FLOOR_DENSE_AM, cuda, make_inputs, run

pytestmark = pytest.mark.gpu


def check(shape, lm, am, seed=61, ul=None, floors=None):
    """One smoothed call with per-utterance weights against the closed form; `ul` overrides the label lengths."""
    N, T, U, V, blank = shape
    trans, pred, labels, tl, ul_ = make_inputs(seed, N, T, U, V, blank)
    ul = ul_ if ul is None else np.asarray(ul, np.int32)
    w = np.linspace(0.5, 1.5, N)
    costs, dF, dG = run(trans, pred, labels, tl, ul, blank, lm, am, w)
    c_ref, dF_ref, dG_ref = sr.closed_form(trans, pred, labels, tl, ul, lm, am, blank, scale=w)
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, **tolerance(am, floors))


def tolerance(am, floors=None):
    """The floors of joint_reference, FLOOR_DENSE_AM on the dense columns when am > 0, and a shape's own floors
    where they are larger."""
    kw = {"floor_dense": FLOOR_DENSE_AM if am > 0 else FLOOR_DENSE, "floor_sparse": FLOOR_SPARSE}
    for k, v in (floors or {}).items():
        kw[k] = max(v, kw[k])
    return kw


# ---- the plain joint's boundary shapes, smoothed --------------------------------------------------------------------
# (0.25, 0.1): every smoothing term; (0.5, 0): no am-only term, so no dF smoothing term and no batch sums.
# A shape keeps the plain joint's floor override (test_gpu_add_joint_geometry.FLOORS): the full term is that joint.
PLAIN_SCALES = [(0.25, 0.1), (0.5, 0.0)]
# Shapes and scales whose data need more, measured on an H100 80GB HBM3 at 700 W:
PLAIN_FLOORS = {
    # 129 frames: Eg / (M sg) (h - hbar) on dG's dense columns is a small difference of two sums over the frames'
    # occupancies; measured floor 1.9e-7 (dG[0] row 13)
    ("T129_second_M_tile_of_1_row", 0.25, 0.1): dict(floor_dense=3e-7),
    # 8 frames for 200 label positions: dF's blank / label columns subtract occupancy totals over 200 positions;
    # measured floor 2.71e-6 (dF[0] row 4, a label column)
    ("U200_V130_two_N_tiles_MODE0", 0.25, 0.1): dict(floor_sparse=4e-6),
}


@pytest.mark.parametrize("lm,am", PLAIN_SCALES)
@pytest.mark.parametrize("name", list(geo.SHAPES))
def test_plain_boundary_shape_smoothed(name, lm, am):
    floors = dict(geo.FLOORS.get(name, {}))
    floors.update(PLAIN_FLOORS.get((name, lm, am), {}))
    check(geo.SHAPES[name], lm, am, floors=floors)


# ---- the smoothing kernels' own boundaries --------------------------------------------------------------------------
# (N, T, U, V, blank, label lengths or None for make_inputs' ragged ones)
SMOOTH_SHAPES = {
    # smooth_chunks: 1 chunk of 32 rows, 2 chunks (17 + 16), 128 chunks of 32, 128 chunks of 33 (the last of 5):
    # over N*U for ug (joint_colsum_kernel<true>) ...
    "NU32_one_chunk": (4, 10, 8, 40, 0, None),
    "NU33_two_chunks": (3, 10, 11, 40, 1, None),
    "NU4096_128_full_chunks": (64, 3, 64, 40, 0, None),
    "NU4097_128_chunks_last_short": (17, 3, 241, 40, 0, None),
    # ... and over N*T for h (joint_colsum_kernel<false>)
    "NT32_one_chunk": (4, 8, 5, 40, 0, None),
    "NT33_two_chunks": (3, 11, 5, 40, 1, None),
    "NT4096_128_full_chunks": (32, 128, 4, 40, 0, None),
    "NT4097_128_chunks_last_short": (17, 241, 4, 40, 0, None),
    # 4800 pred rows in 128 chunks of 38: with U_b = 1 on all but the first utterance, most chunks hold no valid row
    "NU4800_chunks_all_padding": (40, 6, 120, 64, 0, [119] + [0] * 39),
    # the 256-column CTAs of joint_colsum_kernel, joint_unigram_kernel and joint_unigram_grad_kernel
    "V255_one_cta_short": (3, 20, 7, 255, 0, None),
    "V256_one_full_cta": (3, 20, 7, 256, 0, None),
    "V257_second_cta_of_1": (3, 20, 7, 257, 0, None),
    "V513_third_cta_of_1": (3, 20, 7, 513, 2, None),
    # joint_unigram_grad_kernel's shared-memory tiles of 256 (b, u) items: one full tile, a second tile of 1 item
    "NU256_one_item_tile": (8, 10, 32, 50, 0, None),
    "NU257_second_item_tile": (1, 10, 257, 50, 0, None),
    # joint_smooth_rows_kernel: U_b > 32 (a frame row's lanes loop over u) and T_b > 32 (a label row's over t)
    "rows_kernel_Tb70_Ub40": (2, 70, 40, 64, 0, [39, 35]),
    # joint_smooth_g_kernel: hbar over V < 32 (idle lanes), 31 and 33 columns
    "g_kernel_V5": (3, 12, 6, 5, 0, None),
    "g_kernel_V31": (3, 12, 6, 31, 1, None),
    "g_kernel_V33": (3, 12, 6, 33, 0, None),
    # every label_len = 0 (so U = 1): M = N valid pred rows, no label terms anywhere
    "all_label_len_0": (4, 15, 1, 30, 0, [0, 0, 0, 0]),
}
# Measured on an H100 80GB HBM3 at 700 W.  On these the lattice is long in one direction only, so a frame's or a
# label position's occupancy total (O_t, O_u, or the sums of Bk / Lb the blank and label columns subtract) is far
# above 1, and the blank / label columns are small differences of such totals: the fp32 lattice's relative error
# is multiplied by them.
SMOOTH_FLOORS = {
    # 3 frames for up to 241 label positions (O_t ~ 80): measured blank/label floor 5.17e-6 on dF
    ("NU4097_128_chunks_last_short", 0.25, 0.1): dict(floor_sparse=8e-6),
    # the same at c = 0.75 with the am-only term alone: measured 2.1e-5 on dF
    ("NU4097_128_chunks_last_short", 0.0, 0.25): dict(floor_sparse=3e-5),
    # up to 241 frames for 4 label positions: measured 2.57e-6 on dG
    ("NT4097_128_chunks_last_short", 0.0, 0.25): dict(floor_sparse=4e-6),
    # 70 frames and 40 label positions: measured 3.3e-6 on dF and 1.34e-5 on dG (the blank column at 1.125)
    ("rows_kernel_Tb70_Ub40", 0.0, 0.25): dict(floor_sparse=2e-5),
    # measured 1.02e-7 on dG's dense columns
    ("V257_second_cta_of_1", 0.0, 0.25): dict(floor_dense=1.5e-7),
}


@pytest.mark.parametrize("lm,am", [(0.25, 0.1), (0.0, 0.25)])
@pytest.mark.parametrize("name", list(SMOOTH_SHAPES))
def test_smoothing_boundary_shape(name, lm, am):
    *shape, ul = SMOOTH_SHAPES[name]
    check(tuple(shape), lm, am, ul=ul, floors=SMOOTH_FLOORS.get((name, lm, am)))


# ---- training shapes ------------------------------------------------------------------------------------------------
TRAINING = {"C3": (128, 150, 21, 5000), "long": (32, 500, 151, 500)}
# Relative bounds of the sum rules (rows of dF, rows of dG, the column difference) and floor overrides.  C3 keeps
# test_headline_shape's bounds (measured 7.6e-6, 3.4e-6, 4.7e-6 on an H100 80GB HBM3 at 700 W).  At long (T 500,
# U 151, V 500) a row of dF sums to sum_u Wm (S_exact - S) / S: the relative error of S, weighted by the frame's
# occupancy, against a row magnitude that is small where the model already predicts the blank (0.025 at worst).  S
# sums 500 columns in one slab and accumulates stage-wise (DESIGN.md §4); measured on an H100 80GB HBM3 at 400 W,
# largest over (0.25, 0) and (0.25, 0.1): rows of dF 1.58e-5, rows of dG 4.8e-6, columns 9.2e-6 (before the
# stage-wise accumulation: 4.1e-4, 7.2e-6, 2.4e-5 under bounds of 6e-4, 1.5e-5, 4e-5).
SUM_RULES = {"C3": (3e-5, 1e-5, 1e-5), "long": (3e-5, 1e-5, 2e-5)}
# Long needs no override any more (measured dF blank/label floor 1.59e-6 at (0.25, 0), 1.23e-6 at (0.25, 0.1); dG
# within 1e-9 on the dense columns); it needed (1.5e-4, 1.5e-3) and (1.5e-5, 8e-5) before.
TRAINING_FLOORS = {
    ("C3", 0.25, 0.0): dict(floor_sparse=3e-6),                           # measured 2.04e-6 (dF)
}


@pytest.mark.parametrize("lm,am", [(0.25, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("name", list(TRAINING))
def test_training_shape(name, lm, am):
    """Ragged act_len on every third utterance from the second, ragged label_len on every third from the third.
    Every cost and every utterance's gradients against the closed form, determinism, and the sum rules."""
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    N, T, U, V = TRAINING[name]
    blank = 0
    rng = np.random.default_rng(67)
    tl = np.full(N, T, np.int32)
    ul = np.full(N, U - 1, np.int32)
    tl[1::3] = rng.integers(T // 2, T, size=len(tl[1::3]))
    ul[2::3] = rng.integers(0, U - 1, size=len(ul[2::3]))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    gen = torch.Generator("cuda").manual_seed(67)
    trans = torch.randn(N, T, V, device="cuda", generator=gen) * 2
    pred = torch.randn(N, U, V, device="cuda", generator=gen) * 2
    lab, tld, uld = cuda(labels, tl, ul)
    w = torch.linspace(0.5, 1.5, N, device="cuda")

    def step():
        tt, pp = trans.clone().requires_grad_(), pred.clone().requires_grad_()
        out = add_joint_rnnt_loss(tt, pp, lab, tld, uld, blank, 'none', lm_only_scale=lm, am_only_scale=am)
        (out * w).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), tt.grad, pp.grad

    costs, dF, dG = step()
    again = step()
    assert all(torch.equal(a, b) for a, b in zip((costs, dF, dG), again))
    del again

    # sum rules in float64, relative to the sum of |terms| (SUM_RULES).  Rows: each of the three terms' factor
    # gradients sums to 0 over v (a softmax, or for the path through ug Eg / sg (h - hbar)), so every row of dF and
    # dG does.  Columns: the full term's column sums are the same in both factors, so sum_t dF[b,t,v] -
    # sum_u dG[b,u,v] is the difference of the smoothing terms alone, and must be the closed form's.
    rows_f, rows_g, cols = SUM_RULES[name]
    dF64, dG64 = dF.double(), dG.double()
    for x, rtol in ((dF64, rows_f), (dG64, rows_g)):
        excess = x.sum(-1).abs() - rtol * x.abs().sum(-1)
        assert bool((excess <= 0).all()), float(excess.max())
    col, col_mag = (dF64.sum(1) - dG64.sum(1)).cpu().numpy(), (dF64.abs().sum(1) + dG64.abs().sum(1)).cpu().numpy()
    del dF64, dG64

    tr, pr = trans.cpu().numpy(), pred.cpu().numpy()
    c_ref, dF_ref, dG_ref = sr.closed_form(tr, pr, labels, tl, ul, lm, am, blank, scale=w.cpu().numpy())
    excess = np.abs(col - (dF_ref.sum(1) - dG_ref.sum(1))) - cols * col_mag
    assert (excess <= 0).all(), excess.max()
    assert_joint_close(costs.cpu().numpy(), dF.cpu().numpy(), dG.cpu().numpy(), c_ref, dF_ref, dG_ref, labels, tl,
                       ul, blank, **tolerance(am, TRAINING_FLOORS.get((name, lm, am))))


# ---- non-finite padding -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fill", [float("nan"), float("inf"), float("-inf")], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("shape", [(3, 40, 9, 1024, 0), (2, 20, 40, 67, 1)], ids=["fused", "two_kernel"])
def test_non_finite_padding_is_not_read(shape, lm, am, fill):
    """Padded trans frames (t >= act_len) and padded pred rows (u > label_len) hold NaN or +-inf: the costs and the
    valid gradient rows are those of zero padding bit for bit, the padded gradient rows exactly 0.  The fused shape
    runs joint_prep_row_kernel and grad_fused_kernel, the two-kernel shape the warp prep kernel and gemm_kernel."""
    N, T, U, V, blank = shape
    trans, pred, labels, tl, ul = make_inputs(71, N, T, U, V, blank, garbage=False)
    tl[1], ul[1] = T - 7, U // 2   # both factors of utterance 1 padded
    for b in range(N):
        trans[b, tl[b]:] = 0.0
        pred[b, ul[b] + 1:] = 0.0
    clean = run(trans, pred, labels, tl, ul, blank, lm, am)
    for b in range(N):
        trans[b, tl[b]:] = fill
        pred[b, ul[b] + 1:] = fill
    dirty = run(trans, pred, labels, tl, ul, blank, lm, am)
    assert np.array_equal(dirty[0], clean[0]), (dirty[0], clean[0])
    for b in range(N):
        Tb, Ub = int(tl[b]), int(ul[b]) + 1
        assert np.array_equal(dirty[1][b, :Tb], clean[1][b, :Tb]), ("dF", b)
        assert np.array_equal(dirty[2][b, :Ub], clean[2][b, :Ub]), ("dG", b)
        assert not dirty[1][b, Tb:].any() and not dirty[2][b, Ub:].any(), ("padded rows", b)
