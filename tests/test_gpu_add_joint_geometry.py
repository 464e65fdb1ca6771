"""Additive joint (AddJointRNNTLoss) at the boundaries of its dispatch (rnnt_entry.cu run_add_joint) and of the
tensor-core contractions' tiles, slabs and chunks (rnnt_wgmma.cuh), against the fp64 oracle on the
materialised logits (tests/joint_reference.py).

    S = Ef Eg^T   gemm_kernel, M = t in 128-row tiles, N = u in tiles of at most 128, K = v in split-K slabs
    fused grad    grad_fused_kernel (U <= 32): 128-row vocabulary tiles, time in chunks of 32 frames
    dF, dG        gemm_kernel (U > 32): M = v, N = t (64-wide tiles) / N = u, K = u / K = t
    J1 prep       joint_prep_row_kernel<NV> (V % 4 == 0, 1024 <= V <= 8192, aligned rows), else the warp kernel
"""
import numpy as np
import pytest
import torch

from joint_reference import assert_joint_close, reference

pytestmark = pytest.mark.gpu


def make_inputs(seed, N, T, U, V, blank, scale=2.0):
    rng = np.random.default_rng(seed)
    trans = (rng.standard_normal((N, T, V)) * scale).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * scale).astype(np.float32)
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 0))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return trans, pred, labels, tl, ul


def run_joint(trans, pred, labels, tl, ul, blank, weights=None):
    """AddJointRNNTLoss(reduction='none') forward, then backward of sum(costs * weights)."""
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N = trans.shape[0]
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab = torch.as_tensor(labels if labels.size else np.zeros((N, 0), np.int32)).cuda()
    out = AddJointRNNTLoss(blank=blank, reduction='none')(tt, pp, lab, torch.as_tensor(tl).cuda(),
                                                          torch.as_tensor(ul).cuda())
    w = torch.ones(N, device="cuda") if weights is None else torch.as_tensor(weights, dtype=torch.float32).cuda()
    (out * w).sum().backward()
    return out.detach().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy()


def check_shape(shape, seed=41, **floors):
    N, T, U, V, blank = shape
    trans, pred, labels, tl, ul = make_inputs(seed, N, T, U, V, blank)
    w = np.linspace(0.5, 1.5, N)
    costs, dF, dG = run_joint(trans, pred, labels, tl, ul, blank, w)
    c_ref, dF_ref, dG_ref = reference(trans, pred, labels, tl, ul, blank)
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, scale=w, **floors)


# (N, T, U, V, blank): the boundary each shape puts a kernel on
SHAPES = {
    # S: M tiles of 128 frames; the fused gradient's 32-frame chunks; 5 vocabulary tiles (the last with 8 rows)
    "T128_one_full_M_tile": (2, 128, 20, 520, 0),
    "T129_second_M_tile_of_1_row": (2, 129, 20, 520, 3),     # fused: 5 chunks, the last of 1 frame
    "T300_three_M_tiles_U32": (1, 300, 32, 520, 0),          # 3rd M tile 44 rows; 32 label positions (fused limit)
    # S: N = u tiles (64 < U <= 128: one 128-wide tile; U > 128: two tiles), MODE 2 (V % 4 == 0) / MODE 1;
    # dG: 128-wide and two N tiles, MODE 3 / MODE 0 operands; dF: MODE 3 / MODE 0
    "U65_V64_S_128wide_MODE2": (2, 12, 65, 64, 0),
    "U65_V130_S_128wide_MODE1": (2, 12, 65, 130, 1),
    "U128_V64_one_full_N_tile": (2, 10, 128, 64, 0),
    "U128_V130_one_full_N_tile_MODE1": (2, 10, 128, 130, 2),
    "U129_V64_second_N_tile_of_1": (2, 9, 129, 64, 0),
    "U129_V130_second_N_tile_of_1_MODE1": (2, 9, 129, 130, 0),
    "U200_V64_two_N_tiles": (1, 8, 200, 64, 5),
    "U200_V130_two_N_tiles_MODE0": (1, 8, 200, 130, 0),
    # fused gradient: chunk boundaries; V = 129: two vocabulary tiles, the last of 1 row
    "T32_fused_one_full_chunk_V129": (2, 32, 20, 129, 0),
    "T33_fused_two_chunks_U32_V129": (2, 33, 32, 129, 5),
    "T1500_fused_47_chunks_V129": (1, 1500, 24, 129, 0),
    # two-kernel gradient: dG with K = T = 1000; dF with N = T = 1000 in 16 tiles of 64, MODE 3
    "U40_T1000_long_K_dG_16_dF_tiles": (1, 1000, 40, 64, 0),
    # S with both M and N tiled: 3 M tiles of frames (the last of 4 rows) x 2 N tiles of label positions (128 + 23)
    "S_T260_U151_M_and_N_tiled": (1, 260, 151, 132, 0),
    # S split-K: V // 320 slabs (at most 16) of kper = ceil(V / slabs) rounded up to 32
    "V636_one_slab_K636_MODE2": (2, 20, 6, 636, 0),          # the largest V of one slab: 20 stages, the last of 28
    "V641_MODE1_two_slabs": (2, 20, 6, 641, 0),
    "V5001_MODE1_15_slabs": (2, 20, 6, 5001, 4),
    "V5120_exactly_16_slabs": (2, 20, 6, 5120, 0),
    "V5121_MODE1_empty_last_slab": (2, 20, 6, 5121, 0),     # kper 352: slab 15 starts at 5280 > V
    "V5124_MODE2_empty_last_slab": (2, 20, 6, 5124, 7),
    # J1 prep: joint_prep_row_kernel<NV> with NV = ceil(V / 1024) float4 per thread, else the warp kernel
    "V1024_prep_row_1": (2, 10, 5, 1024, 0),
    "V1028_prep_row_2": (2, 10, 5, 1028, 0),
    "V4096_prep_row_4": (2, 10, 5, 4096, 0),
    "V8192_prep_row_8_16_slabs": (2, 10, 5, 8192, 3),
    "V8196_prep_warp_fallback": (2, 10, 5, 8196, 0),
}
# two-kernel gradient (U > 32) over several 128-row vocabulary tiles with V % 4 == 0 (MODE 3 Eg / Ef operands):
# V = 132 (2 tiles, the last of 4 rows), 256 (2 full), 500 (4, the last of 116), 516 (5, the last of 4), crossed with
# K = U = 49, 73, 151 of dF (3, 4 and 7 stages of 24, the last holding 1, 1 and 7 label positions); 136 frames are
# three 64-wide dF tiles, the last of 8.  V = 501: the MODE 0 twins (and S on MODE 1 operands).
for _V in (132, 256, 500, 516, 501):
    for _U, _stages in ((49, 3), (73, 4), (151, 7)):
        SHAPES["V%d_U%d_two_kernel_%d_K_stages%s" % (_V, _U, _stages, "_MODE0" if _V % 4 else "")] = \
            (2, 136, _U, _V, _U % 5)


# Shapes whose data need more than the default floors of tests/joint_reference.py, measured on an H100 80GB HBM3:
FLOORS = {
    # a label column of utterance 1 (weight 1.5), where the dense term and the label terms cancel: measured floor
    # 2.32e-6 on the blank/label columns (|g - g_ref| = 6.3e-6 at g = 0.0402); the tf32 split keeps ~2^-20 per operand
    "T129_second_M_tile_of_1_row": dict(floor_sparse=3e-6),
    # a 1500-frame fp32 lattice: the occupancies' relative error grows with the path length; measured floor
    # 4.52e-9 on the dense columns (relative error 1.2e-4 at g = 1.9e-4)
    "T1500_fused_47_chunks_V129": dict(floor_dense=1e-8),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_joint_boundary_shape(name):
    check_shape(SHAPES[name], **FLOORS.get(name, {}))


def test_plain_joint_long_every_utterance():
    """The long training shape (N 32, T 500, U 151, V 500: S in one slab of K = 500, dF over K = 151 label positions
    in 7 stages, dG over K = 500 frames), ragged act_len on every third utterance from the second and label_len on
    every third from the third.  Every utterance's cost and gradients against smoothed_reference.closed_form at
    scales (0, 0), the plain joint's fp64 reference in closed form (it never forms [T, U, V]), with the default floors."""
    import smoothed_reference as sr
    N, T, U, V, blank = 32, 500, 151, 500, 0
    rng = np.random.default_rng(67)
    tl = np.full(N, T, np.int32)
    ul = np.full(N, U - 1, np.int32)
    tl[1::3] = rng.integers(T // 2, T, size=len(tl[1::3]))
    ul[2::3] = rng.integers(0, U - 1, size=len(ul[2::3]))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    trans = (rng.standard_normal((N, T, V)) * 2).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * 2).astype(np.float32)
    w = np.linspace(0.5, 1.5, N)
    costs, dF, dG = run_joint(trans, pred, labels, tl, ul, blank, w)
    c_ref, dF_ref, dG_ref = sr.closed_form(trans, pred, labels, tl, ul, 0.0, 0.0, blank)
    # cost within 3e-7 relative: measured 1.69e-7 on an H100 80GB HBM3 at 400 W (2.9e-6 when S summed its 500
    # columns in one accumulator, DESIGN.md §4; 8.3e-8 with the SIMT contractions)
    rel = np.abs(costs - c_ref) / np.abs(c_ref)
    assert rel.max() <= 3e-7, rel.max()
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank, scale=w)


def test_misaligned_factors_fall_back_and_match():
    """trans / pred as contiguous views 4 bytes into a larger buffer: the prep falls back from the row kernel
    (16-byte loads) to the warp kernel; the result equals the aligned call bit for bit."""
    from warprnnt_pytorch.joint import add_joint_call
    N, T, U, V, blank = 2, 24, 6, 1024, 0
    trans, pred, labels, tl, ul = make_inputs(43, N, T, U, V, blank)
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))

    def call(tt, pp):
        costs = torch.empty(N, device="cuda")
        dF, dG = torch.full((N, T, V), float("nan"), device="cuda"), torch.full((N, U, V), float("nan"), device="cuda")
        add_joint_call(tt, pp, lab, tld, uld, costs, dF, dG, blank, 1.0)
        torch.cuda.synchronize()
        return costs.cpu().numpy(), dF.cpu().numpy(), dG.cpu().numpy()

    aligned = call(torch.tensor(trans, device="cuda"), torch.tensor(pred, device="cuda"))
    bt = torch.zeros(trans.size + 1, device="cuda")
    bp = torch.zeros(pred.size + 1, device="cuda")
    tt, pp = bt[1:].view(N, T, V), bp[1:].view(N, U, V)
    tt.copy_(torch.as_tensor(trans))
    pp.copy_(torch.as_tensor(pred))
    assert tt.is_contiguous() and tt.data_ptr() % 16 == 4 and pp.data_ptr() % 16 == 4
    shifted = call(tt, pp)
    for a, s in zip(aligned, shifted):
        assert np.array_equal(a, s)
    c_ref, dF_ref, dG_ref = reference(trans, pred, labels, tl, ul, blank)
    assert_joint_close(*shifted, c_ref, dF_ref, dG_ref, labels, tl, ul, blank)


@pytest.mark.parametrize("shape", [(2, 70, 21, 520, 0), (2, 40, 40, 64, 3)], ids=["fused", "two_kernel"])
def test_masked_vocabulary_columns(shape):
    """Columns of trans at -inf (neither the blank nor a label): their gradients are exactly 0 in both
    factors, everything else matches the oracle."""
    N, T, U, V, blank = shape
    trans, pred, labels, tl, ul = make_inputs(47, N, T, U, V, blank)
    used = {blank} | set(labels.reshape(-1).tolist())
    free = np.array([k for k in range(V) if k not in used])
    masked = free[:: max(1, len(free) // 7)]
    assert len(masked) >= 3
    trans[:, :, masked] = -np.inf
    costs, dF, dG = run_joint(trans, pred, labels, tl, ul, blank)
    assert np.all(dF[:, :, masked] == 0) and np.all(dG[:, :, masked] == 0)
    c_ref, dF_ref, dG_ref = reference(trans, pred, labels, tl, ul, blank)
    assert np.all(np.isfinite(costs))
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank)


@pytest.mark.parametrize("shape", [(2, 40, 12, 520, 0), (2, 30, 40, 64, 0)], ids=["fused", "two_kernel"])
def test_wide_dynamic_range_inside_the_fp32_limit(shape):
    """max_v(f+g) about 60 nats below mf+mg (the documented fp32 limit is ~85 nats, rnnt_joint.cuh): trans
    peaks on the first half of the vocabulary, pred on the second, so S = sum_v Ef Eg is ~V e^-60."""
    N, T, U, V, blank = shape
    trans, pred, labels, tl, ul = make_inputs(53, N, T, U, V, blank, scale=0.5)
    half = V // 2
    trans[:, :, :half] += 60.0
    pred[:, :, half:] += 60.0
    gap = (trans.max(-1)[:, :, None] + pred.max(-1)[:, None, :]) - \
        (trans[:, :, None, :] + pred[:, None, :, :]).max(-1)
    assert 55.0 < gap.min() and gap.max() < 65.0
    costs, dF, dG = run_joint(trans, pred, labels, tl, ul, blank)
    c_ref, dF_ref, dG_ref = reference(trans, pred, labels, tl, ul, blank)
    assert_joint_close(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, blank)


def test_headline_shape():
    """N=128, T=150, U=21, V=5000 (the benchmark's C3 shape: S has a second M tile of 22 rows), ragged lengths
    on every third utterance.  Costs of every utterance against the dense RNNTLoss on its materialised logits,
    gradients of four utterances against the oracle, sum rules of dF / dG over the whole batch, determinism."""
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N, T, U, V, blank = 128, 150, 21, 5000, 0
    rng = np.random.default_rng(59)
    tl = np.full(N, T, np.int32)
    ul = np.full(N, U - 1, np.int32)
    tl[1::3] = rng.integers(T // 2, T, size=len(tl[1::3]))
    ul[2::3] = rng.integers(0, U - 1, size=len(ul[2::3]))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    gen = torch.Generator("cuda").manual_seed(59)
    trans = torch.randn(N, T, V, device="cuda", generator=gen) * 2
    pred = torch.randn(N, U, V, device="cuda", generator=gen) * 2
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))
    w = torch.linspace(0.5, 1.5, N, device="cuda")

    def step():
        tt, pp = trans.clone().requires_grad_(), pred.clone().requires_grad_()
        out = AddJointRNNTLoss(blank=blank, reduction='none')(tt, pp, lab, tld, uld)
        (out * w).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), tt.grad, pp.grad

    costs, dF, dG = step()
    again = step()
    assert all(torch.equal(a, b) for a, b in zip((costs, dF, dG), again))
    del again

    dense = RNNTLoss(blank=blank, reduction='none')
    for b in range(N):
        Tb, Ub = int(tl[b]), int(ul[b]) + 1   # the dense operator takes T and U from the longest utterance
        acts = (trans[b:b + 1, :Tb, None, :] + pred[b:b + 1, None, :Ub, :]).contiguous()
        c = dense(acts, lab[b:b + 1, :Ub - 1].contiguous(), tld[b:b + 1], uld[b:b + 1])
        assert np.allclose(costs[b].item(), c.item(), rtol=1e-5), (b, costs[b].item(), c.item())
    del acts

    # utterance 1 has a ragged act_len, utterance 2 a ragged label_len
    pick = [0, 1, int(np.flatnonzero(ul < U - 1)[0]), N - 1]
    assert tl[1] < T and pick[2] == 2
    tr, pr = trans[pick].cpu().numpy(), pred[pick].cpu().numpy()
    c_ref, dF_ref, dG_ref = reference(tr, pr, labels[pick], tl[pick], ul[pick], blank)
    assert_joint_close(costs[pick].cpu().numpy(), dF[pick].cpu().numpy(), dG[pick].cpu().numpy(), c_ref, dF_ref,
                       dG_ref, labels, tl, ul, blank, batch=pick, scale=w[pick].cpu().numpy())
    del dF_ref, dG_ref

    # sum rules over the whole batch, in float64: every logit's gradient sums to 0 over v (softmax), so each row
    # of dF and dG does; both factors' column sums equal sum_{t,u} dL/dh[b,t,u,v].  Relative to the sum of
    # |terms|; largest ratio measured on an H100 80GB HBM3: rows of dF 1.15e-5 (one frame's row sums over up to
    # 21 label positions and 5000 columns), rows of dG 4.4e-6, columns 3.5e-6.
    dF64, dG64 = dF.double(), dG.double()
    for x, rtol in ((dF64, 3e-5), (dG64, 1e-5)):
        excess = x.sum(-1).abs() - rtol * x.abs().sum(-1)
        assert bool((excess <= 0).all()), float(excess.max())
    excess = (dF64.sum(1) - dG64.sum(1)).abs() - 1e-5 * (dF64.abs().sum(1) + dG64.abs().sum(1))
    assert bool((excess <= 0).all()), float(excess.max())
