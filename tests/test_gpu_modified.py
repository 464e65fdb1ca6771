"""The modified (one symbol per frame) topology (DESIGN.md §11) on the GPU against the fp64 reference
(tests/modified_reference.py).

Bars (§6): costs 1e-5 relative, gradients 1e-4 relative + 1e-6 absolute; with a delay penalty the cost bar is
1e-5 * max(|cost|, 1 + lambda T_b U_b / 2), as §10 scales it.  fp64 uses 1e-11 on costs and 1e-9 relative on
gradients; 16-bit storage is compared with the reference on the rounded logits, gradients to the storage type's
rounding.  An utterance without a path must cost +inf with an all-zero gradient."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import modified_reference as mr
import pruned_reference as pr
from test_gpu_delay_penalty import (STORAGES, TORCH, assert_joint, cost_bar, cuda, f32, grad_tol, joint_inputs,
                                    make)
from test_gpu_tuning_hooks import norm

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
# (N, T, U, V): the dispatch family / wavefront each shape reaches for fp32 (16-bit rows are half as long).  T >= U - 1
# so that most utterances have a path; make() keeps utterance 0 at T, U - 1.
SHAPES = {
    "chunk": (4, 12, 6, 28),              # rows <= 512 B: grad_chunk_mod_kernel; single-warp wavefront, 1 column
    "tile": (3, 10, 5, 500),              # register tiles
    "row": (2, 6, 4, 1500),               # one CTA per row
    "cols2_U40": (3, 45, 40, 20),         # fp32 wavefront with two columns per lane; fp64 multi-warp
    "cols2_U64": (2, 70, 64, 12),         # two columns per lane, the last lane's pair full
    "wavefront_U65": (2, 70, 65, 20),     # multi-warp fp32 wavefront (one column per lane), 3 warps
    "wavefront_U301": (2, 310, 301, 8),   # 10 warps
}

def run_operator(acts_np, labels, tl, ul, storage, weights=None, **kw):
    """rnnt_loss(reduction='none', rnnt_type='modified') forward + backward with per-utterance grad_output."""
    from warprnnt_pytorch import rnnt_loss
    x = torch.tensor(acts_np, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = rnnt_loss(x, lab, tl_, ul_, reduction='none', rnnt_type='modified', **kw)
    w = torch.ones_like(out) if weights is None else torch.as_tensor(weights).to(out)
    w = torch.where(torch.isfinite(out), w, torch.zeros_like(w))   # no NaN from inf * 0 in autograd's sum
    (torch.where(torch.isfinite(out), out, torch.zeros_like(out)) * w).sum().backward()
    torch.cuda.synchronize()
    used = x.detach().double().cpu().numpy()      # the logits as stored (16-bit: rounded)
    return out.detach().double().cpu().numpy(), x.grad.double().cpu().numpy(), used


def assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage):
    fin = np.isfinite(c_ref)
    assert np.array_equal(np.isfinite(costs), fin), (costs, c_ref)
    assert (costs[~fin] == np.inf).all()
    assert not grads[~fin].any(), "an utterance without a path has a gradient"
    rel_c = 1e-11 if storage == "fp64" else 1e-5
    err = np.abs(costs[fin] - c_ref[fin])
    bar = cost_bar(c_ref[fin], lam, tl[fin], ul[fin], rel_c)
    assert (err <= bar).all(), (err / bar).max()
    rt, at = grad_tol(storage)
    excess = np.abs(grads - g_ref) - (rt * np.abs(g_ref) + at)
    assert excess.max() <= 0, excess.max()


def mixed(seed, N, T, U, V):
    """make() with T_b >= U_b - 1 except for one utterance without a path (when N > 2)."""
    acts, labels, tl, ul = make(seed, N, T, U, V)
    ul[1:] = np.minimum(ul[1:], tl[1:])
    if N > 2:
        tl[N - 1], ul[N - 1] = max(1, min(T, U - 2) // 2), min(U - 1, max(1, min(T, U - 2) // 2) + 1)
        assert ul[N - 1] > tl[N - 1]
    return acts, labels, tl, ul


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_against_reference(shape, storage):
    N, T, U, V = SHAPES[shape]
    acts, labels, tl, ul = mixed(1, N, T, U, V)
    w = np.linspace(0.5, 1.5, N)
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, w)
    c_ref, g_ref = mr.dense_loss(used, labels, tl, ul)
    assert_close(costs, grads, c_ref, g_ref * w[:, None, None, None], 0.0, tl, ul, storage)


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("T,U", [(1, 1), (1, 2), (5, 1), (7, 8), (40, 41), (70, 65), (3, 9)],
                         ids=lambda v: str(v))
def test_edge_extents(T, U, storage):
    """T = 1, U = 1, T_b = U_b - 1 (a single path: every frame a label) and no path at all, every utterance full."""
    N, V = 2, 20
    acts, labels, tl, ul = make(2, N, T, U, V)
    tl[:], ul[:] = T, U - 1
    costs, grads, used = run_operator(acts, labels, tl, ul, storage)
    c_ref, g_ref = mr.dense_loss(used, labels, tl, ul)
    assert_close(costs, grads, c_ref, g_ref, 0.0, tl, ul, storage)


@pytest.mark.parametrize("storage", STORAGES)
def test_fastemit_clamp_and_delay_penalty(storage):
    N, T, U, V = SHAPES["tile"]
    acts, labels, tl, ul = mixed(3, N, T, U, V)
    for lam, fe, clamp in ((0.4, 0.0, -1.0), (0.0, 0.3, -1.0), (0.0, 0.0, 0.015625), (0.4, 0.3, 0.015625)):
        costs, grads, used = run_operator(acts, labels, tl, ul, storage, delay_penalty=f32(lam),
                                          fastemit_lambda=f32(fe), clamp=clamp)
        c_ref, g_ref = mr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam), fastemit_lambda=f32(fe),
                                     clamp=clamp)
        assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage)


@pytest.mark.parametrize("storage", ["fp32", "fp64"])
def test_tunv_layout_split_and_full_call(storage):
    """The full call, [N,T,U,V] and [T,U,N,V], against the forward / backward split with per-utterance grad_output,
    and the reference."""
    from warprnnt_pytorch import warp_rnnt
    N, T, U, V = SHAPES["chunk"]
    acts, labels, tl, ul = mixed(4, N, T, U, V)
    lam = 0.25
    w = np.linspace(0.5, 1.5, N)
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, w, delay_penalty=f32(lam))
    x = torch.tensor(acts, device="cuda", dtype=TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    wd = torch.tensor(np.where(np.isfinite(costs), w, 0.0), device="cuda", dtype=x.dtype)
    c_full = torch.empty(N, device="cuda", dtype=x.dtype)
    g_full = torch.empty_like(x)
    ws = warp_rnnt.gpu_rnnt_async(x, lab, tl_, ul_, c_full, g_full, 0, delay_penalty=f32(lam), rnnt_type='modified')
    xt = x.permute(1, 2, 0, 3).contiguous()
    c_t = torch.empty(N, device="cuda", dtype=x.dtype)
    g_t = torch.empty_like(xt)
    ws2 = warp_rnnt.gpu_rnnt_async_tunv(xt, lab, tl_, ul_, c_t, g_t, 0, delay_penalty=f32(lam), rnnt_type='modified')
    c_s = torch.empty(N, device="cuda", dtype=x.dtype)
    ws3 = warp_rnnt.gpu_rnnt_forward(x, lab, tl_, ul_, c_s, 0, delay_penalty=f32(lam), rnnt_type='modified')
    g_s = torch.full_like(x, float("nan"))
    warp_rnnt.gpu_rnnt_backward(x, lab, tl_, ul_, g_s, wd, 0, 1.0, ws3, delay_penalty=f32(lam), rnnt_type='modified')
    torch.cuda.synchronize()
    del ws, ws2
    assert np.array_equal(c_full.double().cpu().numpy(), costs)
    assert np.array_equal(c_t.double().cpu().numpy(), costs)
    assert np.array_equal(c_s.double().cpu().numpy(), costs)
    assert np.array_equal(g_t.permute(2, 0, 1, 3).double().cpu().numpy(), g_full.double().cpu().numpy())
    assert np.array_equal(g_s.double().cpu().numpy(), grads)
    c_ref, g_ref = mr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam))
    assert_close(costs, grads, c_ref, g_ref * np.where(np.isfinite(c_ref), w, 0.0)[:, None, None, None], lam, tl, ul,
                 storage)
    assert_close(costs, g_full.double().cpu().numpy(), c_ref, g_ref, lam, tl, ul, storage)
    # the forward and backward log-likelihoods the wavefronts left in the workspace agree
    f, b = warp_rnnt.read_log_likelihoods(ws3, T, U, N, 8 if storage == "fp64" else 4)
    fin = np.isfinite(c_ref)
    np.testing.assert_allclose(f[fin], -c_ref[fin], rtol=1e-5 if storage == "fp32" else 1e-11)
    np.testing.assert_allclose(b[fin], f[fin], rtol=1e-5 if storage == "fp32" else 1e-11)
    assert (f[~fin] < -1e8).all() and (b[~fin] < -1e8).all()     # log zero (fp32: an exponent near -2^29)


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", ["chunk", "tile", "wavefront_U65"])
def test_nan_prefilled_gradients_zero_on_padding_and_dead_utterances(storage, shape):
    from warprnnt_pytorch import warp_rnnt
    N, T, U, V = SHAPES[shape]
    N = 3
    acts, labels, tl, ul = mixed(5, N, T, U, V)
    x = torch.tensor(acts, device="cuda").to(TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    costs = torch.empty(N, device="cuda", dtype=warp_rnnt.costs_dtype(x))
    ws = warp_rnnt.gpu_rnnt_forward(x, lab, tl_, ul_, costs, 0, rnnt_type='modified')
    grads = torch.full_like(x, float("nan"))
    warp_rnnt.gpu_rnnt_backward(x, lab, tl_, ul_, grads, None, 0, 1.0, ws, rnnt_type='modified')
    g = grads.double().cpu().numpy()
    c = costs.double().cpu().numpy()
    assert c[N - 1] == np.inf and not g[N - 1].any()
    for b in range(N - 1):
        assert np.isfinite(c[b])
        assert np.isfinite(g[b, :tl[b], :ul[b] + 1]).all()
        assert (g[b, tl[b]:] == 0).all() and (g[b, :, ul[b] + 1:] == 0).all()


def test_regular_through_every_new_path_is_the_existing_entry_bitwise():
    """rnnt_type='regular' through the keyword and rnnt_type = 0 through the *_topo entries compute exactly what
    the existing entries do."""
    from warprnnt_pytorch import rnnt_loss, warp_rnnt
    N, T, U, V = SHAPES["tile"]
    acts, labels, tl, ul = make(6, N, T, U, V)
    for storage in STORAGES:
        x = torch.tensor(acts, device="cuda").to(TORCH[storage]).requires_grad_(True)
        lab, tl_, ul_ = cuda(labels, tl, ul)
        outs = []
        for kw in ({}, {"rnnt_type": "regular"}):
            x.grad = None
            out = rnnt_loss(x, lab, tl_, ul_, reduction='none', delay_penalty=0.25, **kw)
            out.sum().backward()
            outs.append((out.detach().cpu(), x.grad.cpu()))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    lib = warp_rnnt.lib()
    x = torch.tensor(acts, device="cuda")
    lab, tl_, ul_ = cuda(labels, tl, ul)
    opt = warp_rnnt._options(x, 0)
    for lam in (0.0, 0.25):
        res = []
        for topo in (False, True):
            c = torch.empty(N, device="cuda")
            g = torch.empty_like(x)
            ws = torch.empty(warp_rnnt.workspace_size(T, U, N), dtype=torch.uint8, device="cuda")
            args = (0, 0, x.data_ptr(), g.data_ptr(), lab.data_ptr(), ul_.data_ptr(), tl_.data_ptr(), V, N,
                    c.data_ptr(), 1.0, warp_rnnt.rnntGradOptions(0.3, 0.0), warp_rnnt.rnntLatticeOptions(lam))
            st = (lib.rnnt_b200_loss_async_topo(*args, 0, ws.data_ptr(), opt) if topo
                  else lib.rnnt_b200_loss_async_lat(*args, ws.data_ptr(), opt))
            assert st == 0
            c2 = torch.empty(N, device="cuda")
            ws2 = torch.empty_like(ws)
            fargs = (0, x.data_ptr(), lab.data_ptr(), ul_.data_ptr(), tl_.data_ptr(), V, N, c2.data_ptr(), 1,
                     warp_rnnt.rnntLatticeOptions(lam))
            st = (lib.rnnt_b200_forward_topo(*fargs, 0, ws2.data_ptr(), opt) if topo
                  else lib.rnnt_b200_forward_lat(*fargs, ws2.data_ptr(), opt))
            assert st == 0
            g2 = torch.empty_like(x)
            bargs = (0, x.data_ptr(), g2.data_ptr(), lab.data_ptr(), ul_.data_ptr(), tl_.data_ptr(), V, N, None, 0.5,
                     warp_rnnt.rnntGradOptions(0.0, 0.01), warp_rnnt.rnntLatticeOptions(lam))
            st = (lib.rnnt_b200_backward_topo(*bargs, 0, ws2.data_ptr(), opt) if topo
                  else lib.rnnt_b200_backward_lat(*bargs, ws2.data_ptr(), opt))
            assert st == 0
            torch.cuda.synchronize()
            res.append([t.cpu() for t in (c, g, c2, g2)])
        assert all(torch.equal(a, b) for a, b in zip(*res)), lam


# ---- pruned ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", ["chunk", "tile", "wavefront_U65"])
def test_pruned_full_windows_are_the_dense_loss_bitwise(storage, shape):
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, V = SHAPES[shape]
    N = 3
    acts, labels, tl, ul = mixed(7, N, T, U, V)
    lam = 0.3
    costs, grads, _ = run_operator(acts, labels, tl, ul, storage, delay_penalty=f32(lam))
    x = torch.tensor(acts, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    ranges = torch.zeros(N, T, dtype=torch.int32, device="cuda")
    out = pruned_rnnt_loss(x, lab, tl_, ul_, ranges, reduction='none', delay_penalty=f32(lam), rnnt_type='modified')
    torch.where(torch.isfinite(out), out, torch.zeros_like(out)).sum().backward()
    assert np.array_equal(out.detach().double().cpu().numpy(), costs)
    assert np.array_equal(x.grad.double().cpu().numpy(), grads)


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("V", [28, 500])
def test_pruned_against_reference_with_adversarial_windows(storage, V):
    """Random monotone windows (some leave a modified path, some advance faster than one label per frame and do not)
    against the reference."""
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, R = 6, 12, 7, 3
    rng = np.random.default_rng(8)
    _, labels, tl, ul = make(8, N, T, U, 2)
    ul[:] = np.minimum(ul, tl)
    labels = rng.integers(1, V, size=labels.shape).astype(np.int32)
    ranges = pr.random_monotone_ranges(rng, tl, ul, T, R)
    ranges[1, 1:tl[1]] = np.maximum(ranges[1, 1:tl[1]], 2)    # frame 1 starts at u = 2: no modified path
    logits = (rng.standard_normal((N, T, R, V)) * 1.5).astype(np.float32)
    lam = 0.4
    x = torch.tensor(logits, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_, rg = cuda(labels, tl, ul, ranges)
    out = pruned_rnnt_loss(x, lab, tl_, ul_, rg, reduction='none', delay_penalty=f32(lam), fastemit_lambda=0.25,
                           rnnt_type='modified')
    w = torch.linspace(0.5, 1.5, N, device="cuda").to(out)
    w = torch.where(torch.isfinite(out), w, torch.zeros_like(w))
    (torch.where(torch.isfinite(out), out, torch.zeros_like(out)) * w).sum().backward()
    c_ref, g_ref = mr.loss(x.detach().double().cpu().numpy(), labels, tl, ul, ranges, delay_penalty=f32(lam),
                           fastemit_lambda=0.25)
    assert not np.isfinite(c_ref[1]) and np.isfinite(c_ref).any()
    assert_close(out.detach().double().cpu().numpy(), x.grad.double().cpu().numpy(), c_ref,
                 g_ref * w.double().cpu().numpy()[:, None, None, None], lam, tl, ul, storage)


# ---- additive joint ----------------------------------------------------------------------------------------------
def joint_mixed(seed, N, T, U, V):
    trans, pred, labels, tl, ul = joint_inputs(seed, N, T, U, V)
    ul[1:] = np.minimum(ul[1:], tl[1:])
    tl[N - 1], ul[N - 1] = 2, min(U - 1, 4)      # no path
    return trans, pred, labels, tl, ul


def run_joint(trans, pred, labels, tl, ul, lm=0.0, am=0.0, weights=None, **kw):
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = add_joint_rnnt_loss(tt, pp, lab, tl_, ul_, 0, 'none', lm_only_scale=lm, am_only_scale=am,
                              rnnt_type='modified', **kw)
    w = torch.ones_like(out) if weights is None else torch.as_tensor(weights, dtype=torch.float32).cuda()
    (torch.where(torch.isfinite(out), out, torch.zeros_like(out)) * w).sum().backward()
    torch.cuda.synchronize()
    return out.detach().double().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy()


def assert_joint_mod(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, lam, floor_dense=1e-9):
    fin = np.isfinite(c_ref)
    assert np.array_equal(np.isfinite(costs), fin) and (costs[~fin] == np.inf).all(), (costs, c_ref)
    c_ref = np.where(fin, c_ref, 0.0)
    costs = np.where(fin, costs, 0.0)
    assert_joint(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, lam, np.ones(len(tl)), floor_dense)


@pytest.mark.parametrize("shape", [(3, 20, 7, 64), (3, 45, 40, 131), (3, 40, 9, 1024)],
                         ids=lambda s: "N%d_T%d_U%d_V%d" % s)
def test_joint_matches_the_dense_loss_on_materialised_logits(shape):
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N, T, U, V = shape
    trans, pred, labels, tl, ul = joint_mixed(9, N, T, U, V)
    lam = 0.3
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    j = AddJointRNNTLoss(reduction='none', delay_penalty=f32(lam), rnnt_type='modified')(tt, pp, lab, tl_, ul_)
    torch.where(torch.isfinite(j), j, torch.zeros_like(j)).sum().backward()
    acts = (tt.detach().double().unsqueeze(2) + pp.detach().double().unsqueeze(1)).requires_grad_(True)
    d = RNNTLoss(reduction='none', delay_penalty=f32(lam), rnnt_type='modified')(acts, lab, tl_, ul_)   # fp64 dense
    torch.where(torch.isfinite(d), d, torch.zeros_like(d)).sum().backward()
    assert_joint_mod(j.detach().double().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy(),
                     d.detach().cpu().numpy(), acts.grad.sum(2).cpu().numpy(), acts.grad.sum(1).cpu().numpy(),
                     labels, tl, ul, lam)


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("fe,lam", [(0.0, 0.0), (0.3, 0.3)])
def test_joint_against_reference(lm, am, fe, lam):
    N, T, U, V = 3, 24, 8, 131
    trans, pred, labels, tl, ul = joint_mixed(10, N, T, U, V)
    w = np.linspace(0.5, 1.5, N)
    got = run_joint(trans, pred, labels, tl, ul, lm, am, w, fastemit_lambda=f32(fe), delay_penalty=f32(lam))
    want = mr.joint_reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul, lm, am,
                              delay_penalty=f32(lam), fastemit_lambda=f32(fe), scale=w)
    assert_joint_mod(*got, *want, labels, tl, ul, lam, floor_dense=1e-7 if am > 0 else 1e-9)


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0)])
def test_joint_modified_ranges(lm, am):
    """The modified ranges equal the reference's (steps 1-3 on the modified occupancies) and differ from the
    regular ones on the same inputs."""
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    N, T, U, V, R = 4, 30, 9, 64, 3
    for seed in range(20, 80):
        trans, pred, labels, tl, ul = joint_inputs(seed, N, T, U, V)
        ul[:] = np.minimum(ul, tl)
        want, margin = mr.prune_ranges(trans, pred, labels, tl, ul, T, R, lm, am)
        if margin > 1e-4:
            break
    assert margin > 1e-4, "no seed with unambiguous windows"
    tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
    loss, ranges = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, R, reduction='none', lm_only_scale=lm,
                                                   am_only_scale=am, rnnt_type='modified')
    got = ranges.cpu().numpy()
    assert np.array_equal(got, want)
    pr.check_range_properties(got, tl, ul, R)
    c_ref = mr.joint_costs(trans, pred, labels, tl, ul, lm, am)
    assert (np.abs(loss.detach().double().cpu().numpy() - c_ref) <= 1e-5 * np.maximum(np.abs(c_ref), 1.0)).all()
    # a workspace without a path: every inner frame scores 0 and starts at 0
    tl2, ul2 = tl.copy(), ul.copy()
    tl2[1], ul2[1] = 5, 8
    _, r2 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, *cuda(tl2, ul2), R, reduction='none', rnnt_type='modified')
    want2, _ = mr.prune_ranges(trans, pred, labels, tl2, ul2, T, R)
    assert np.array_equal(r2.cpu().numpy(), want2)


def test_joint_regular_through_every_new_path_is_the_existing_entry_bitwise():
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges, warp_rnnt
    from warprnnt_pytorch.joint import _joint_opts, _lab_ptr, _lib, joint_forward_call, rnntSmoothOptions
    N, T, U, V = 3, 20, 7, 64
    trans, pred, labels, tl, ul = joint_inputs(11, N, T, U, V)
    tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
    g = torch.linspace(0.5, 1.5, N, device="cuda")
    for lm, am in ((0.0, 0.0), (0.25, 0.1)):
        smooth = rnntSmoothOptions(lm, am) if lm or am else None
        res = []
        for topo in (None, warp_rnnt.RNNT_B200_RNNT_REGULAR):
            c = torch.empty(N, device="cuda")
            kw = {} if topo is None else {"topo": topo}
            ws = joint_forward_call(tt, pp, lab, tl_, ul_, c, True, 0, smooth, warp_rnnt.rnntLatticeOptions(0.2), **kw)
            dF, dG = torch.empty_like(tt), torch.empty_like(pp)
            args = (tt.data_ptr(), pp.data_ptr(), dF.data_ptr(), dG.data_ptr(), _lab_ptr(lab), ul_.data_ptr(),
                    tl_.data_ptr(), V, N, g.data_ptr(), 0.5, warp_rnnt.rnntGradOptions(0.3, 0.0))
            tail = (ws.data_ptr(), _joint_opts(tt, pp, 0))
            if topo is None:
                st = _lib.rnnt_b200_add_joint_smoothed_backward(*args, smooth or rnntSmoothOptions(), *tail)
            else:
                st = _lib.rnnt_b200_add_joint_backward_topo(*args, smooth or rnntSmoothOptions(), topo, *tail)
            assert st == 0
            ranges = torch.empty(N, T, dtype=torch.int32, device="cuda")
            if topo is None:
                st = _lib.rnnt_b200_add_joint_prune_ranges(ul_.data_ptr(), tl_.data_ptr(), N, 3, ranges.data_ptr(),
                                                           ws.data_ptr(), _joint_opts(tt, pp, 0))
            else:
                st = _lib.rnnt_b200_add_joint_prune_ranges_topo(ul_.data_ptr(), tl_.data_ptr(), N, 3,
                                                                ranges.data_ptr(), ws.data_ptr(), topo,
                                                                _joint_opts(tt, pp, 0))
            assert st == 0
            torch.cuda.synchronize()
            res.append([t.cpu() for t in (c, dF, dG, ranges)])
        assert all(torch.equal(a, b) for a, b in zip(*res)), (lm, am)
        _, r0 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, lm_only_scale=lm, am_only_scale=am)
        _, r1 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, lm_only_scale=lm, am_only_scale=am,
                                                rnnt_type='regular')
        assert torch.equal(r0, r1)


# ---- batch groups and tuning hooks (child processes: the hooks are read once per process) -------------------------
def test_grouped_schedule_is_bitwise_the_ungrouped_call():
    e = dict(os.environ)
    e["RNNT_B200_GROUPS"] = "4"
    r = subprocess.run([sys.executable, os.path.join(HERE, "modified_hook_child.py"), "groups"], env=e,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "groups ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def _hook_cases():
    from test_gpu_tuning_hooks import CASES
    return ["default"] + sorted({tuple(sorted(env.items())) for _, env, _, _, _ in CASES.values()})


# kernels of the regular topology that have a modified twin
REGULAR = re.compile(r"(grad_(chunk|tile|row)(_delay)?_kernel<|lattice_lin_kernel<|lattice_kernel<|"
                     r"joint_weights_kernel<)")
TWINS = ("grad_chunk_mod_kernel<float, 2, 256, false>", "grad_chunk_mod_kernel<float, 2, 256, true>",
         "lattice_lin_mod_kernel<1, false, 8>", "lattice_lin_mod_kernel<1, true, ", "joint_weights_mod_kernel<")


@pytest.mark.parametrize("hook", _hook_cases(), ids=lambda h: h if isinstance(h, str) else
                         "_".join("%s=%s" % (k[len("RNNT_B200_"):], v) for k, v in h))
def test_tuning_hooks(hook):
    """Every hook setting of test_gpu_tuning_hooks.CASES, one process each: the dense, pruned and joint shapes of
    hook_cases.py with rnnt_type='modified' match the reference, and only the modified instantiations of the
    gradient, lattice and joint-weights kernels ran."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("RNNT_B200_")}
    if hook != "default":
        env.update(dict(hook))
    r = subprocess.run([sys.executable, os.path.join(HERE, "modified_hook_child.py"), "hooks"], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    rep = json.loads(r.stdout.strip().splitlines()[-1])
    assert not rep["problems"], rep["problems"]
    kernels = [norm(k) for k in rep["kernels"]]
    assert not [k for k in kernels if REGULAR.search(k)], [k for k in kernels if REGULAR.search(k)]
    assert any("_mod_kernel<" in k for k in kernels)
    if hook == "default":
        for twin in TWINS:
            assert any(twin in k for k in kernels), (twin, [k for k in kernels if "mod" in k])
