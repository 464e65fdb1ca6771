"""The loss, gradient and forced alignment on caller-supplied factors (DESIGN.md §13) on the GPU, against the fp64
reference (tests/lattice_reference.py), rnnt_loss, and the constrained transducer's definition.

Bars (§6, the cost bar scaled as §10 does for costs near zero): costs within 1e-5 * max(|cost|, 1) (fp64 storage:
1e-11), gradients within 1e-4 relative + 1e-6 absolute (fp64: 1e-10 + 1e-12).  The fp32 arithmetic splits each
factor into m 2^k with m from ex2.approx (2 ulp), so a path of n factors carries about n 2^-22 of error in its
log-probability whatever its magnitude: the fp32 bars get n 2^-22 (absolute for costs, relative for gradients), as
§12's do.  16-bit storage is compared with the reference on the rounded factors, and its gradients, written in the
storage type, get one rounding of that type on top."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import align_reference as ar
import lattice_reference as lr
from test_gpu_delay_penalty import STORAGES, TORCH, cuda

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TOPOLOGIES = ["regular", "modified"]
MOD = {"regular": False, "modified": True}
# (N, S, T): maxU = S + 1 covers one to 32 warps of the fp32 wavefront (two columns per lane at 33..64, the cross-warp
# exchange from 65) and of the Viterbi kernel; T = 1 and a long T
SHAPES = {
    "U1": (3, 0, 150),
    "U2": (3, 1, 150),
    "U21": (4, 20, 150),
    "U32": (3, 31, 150),
    "U33": (3, 32, 150),
    "U41": (3, 40, 150),
    "U64": (2, 63, 150),
    "U65": (2, 64, 150),
    "U301": (2, 300, 150),
    "U1024": (2, 1023, 40),
    "T1": (3, 4, 1),
    "T1500": (2, 300, 1500),
}
LONG = {"U1024", "T1500"}   # the fp64 numpy reference takes seconds per utterance here: fp32 and fp64 storage only
ROUND = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}


def factors(seed, N, S, T, topo="regular"):
    """Normalised random factors (a three-way softmax per cell: blank, label, rest) and ragged lengths with
    T == max(T_b), S == max(S_b); modified: S_b <= T_b."""
    rng = np.random.default_rng(seed)
    lp = rng.standard_normal((N, S + 1, T, 3)) * 1.5
    lp -= np.log(np.exp(lp).sum(-1, keepdims=True))
    py, px = lp[..., 0].copy(), lp[:, :S, :, 1].copy()
    tl = rng.integers(max(1, T // 2), T + 1, N).astype(np.int32)
    ul = rng.integers(0, S + 1, N).astype(np.int32)
    tl[0], ul[0] = T, S
    if topo == "modified":
        ul = np.minimum(ul, tl)
        ul[0] = S   # S > T: utterance 0 has more labels than frames, and no path
    return px, py, tl, ul


def seed(shape, topo):
    return 2 * sorted(SHAPES).index(shape) + TOPOLOGIES.index(topo)


def to_dev(px, py, storage, grad=True):
    x = torch.tensor(px, device="cuda").to(TORCH[storage]).requires_grad_(grad)
    y = torch.tensor(py, device="cuda").to(TORCH[storage]).requires_grad_(grad)
    return x, y


def run_loss(px, py, tl, ul, storage, topo, reduction="none", grad_output=None):
    """(costs, px grad, py grad, px and py as stored) in float64 through rnnt_lattice_loss and autograd."""
    from warprnnt_pytorch import rnnt_lattice_loss
    x, y = to_dev(px, py, storage)
    costs = rnnt_lattice_loss(x, y, *cuda(tl, ul), reduction, rnnt_type=topo)
    assert costs.dtype == (torch.float64 if storage == "fp64" else torch.float32)
    costs.backward(torch.ones_like(costs) if grad_output is None else grad_output)
    torch.cuda.synchronize()
    assert x.grad.dtype == TORCH[storage] and y.grad.dtype == TORCH[storage]
    f = lambda t: t.detach().double().cpu().numpy()   # noqa: E731
    return f(costs), f(x.grad), f(y.grad), f(x), f(y)


def n_factors(tl, ul, topo):
    return np.asarray(tl) + (0 if topo == "modified" else np.asarray(ul))


def cost_bar(ref, storage, nf):
    if storage == "fp64":
        return 1e-11 * np.maximum(np.abs(ref), 1.0)
    return 1e-5 * np.maximum(np.abs(ref), 1.0) + nf * 2.0 ** -22


def assert_costs(costs, ref, storage, nf):
    assert np.array_equal(np.isnan(costs), np.isnan(ref)), (costs, ref)
    assert np.array_equal(np.isinf(costs), np.isinf(ref)), (costs, ref)
    assert (costs[np.isinf(ref)] == ref[np.isinf(ref)]).all()
    fin = np.isfinite(ref)
    err = np.abs(costs[fin] - ref[fin])
    assert (err <= cost_bar(ref[fin], storage, nf[fin])).all(), (costs[fin], ref[fin], err)


def assert_grads(g, ref, storage, nf, live):
    """Per utterance b with live[b]; the bars of the module docstring."""
    for b in np.flatnonzero(live):
        if storage == "fp64":
            tol = 1e-10 * np.abs(ref[b]) + 1e-12
        else:
            tol = (1e-4 + nf[b] * 2.0 ** -22 + ROUND.get(storage, 0.0)) * np.abs(ref[b]) + 1e-6
        err = np.abs(g[b] - ref[b])
        assert (err <= tol).all(), (b, err.max(), np.unravel_index(np.argmax(err - tol), err.shape))


def check_against_reference(px, py, tl, ul, storage, topo):
    costs, gx, gy, ux, uy = run_loss(px, py, tl, ul, storage, topo)
    rc, rgx, rgy = lr.loss(ux, uy, tl, ul, MOD[topo])
    nf = n_factors(tl, ul, topo)
    assert_costs(costs, rc, storage, nf)
    live = ~np.isnan(rc)
    assert_grads(gx, rgx, storage, nf, live)
    assert_grads(gy, rgy, storage, nf, live)
    return costs, gx, gy


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_against_reference(shape, storage, topo):
    if shape in LONG and storage in ROUND:
        pytest.skip("long shapes: fp32 and fp64 storage only")
    px, py, tl, ul = factors(seed(shape, topo), *SHAPES[shape], topo=topo)
    check_against_reference(px, py, tl, ul, storage, topo)


@pytest.mark.parametrize("storage", STORAGES)
def test_modified_edges(storage):
    """S_b = 0, S_b = T_b (every frame emits a label) and S_b > T_b (no path: +inf, zero gradient) side by side."""
    px, py, _, _ = factors(3, 4, 7, 6)
    tl = np.array([6, 6, 5, 6], np.int32)
    ul = np.array([6, 0, 7, 3], np.int32)
    costs, gx, gy = check_against_reference(px, py, tl, ul, storage, "modified")
    assert costs[2] == np.inf and not gx[2].any() and not gy[2].any()
    assert np.isfinite(costs[[0, 1, 3]]).all()


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("S,T", [(5, 12), (40, 60), (100, 150)])
def test_minus_inf_factors_and_dead_utterances(S, T, storage, topo):
    """Scattered -inf factors in live utterances, and utterances whose factors leave no path (all blanks -inf; every
    label factor -inf with labels) next to them: +inf with a zero gradient."""
    px, py, tl, ul = factors(S + T, 4, S, T, topo)
    rng = np.random.default_rng(S)
    px[rng.random(px.shape) < 0.2] = -np.inf
    py[0][rng.random(py[0].shape) < 0.1] = -np.inf
    py[1] = -np.inf
    px[2] = -np.inf
    ul[2] = max(ul[2], 1)
    costs, gx, gy = check_against_reference(px, py, tl, ul, storage, topo)
    for b in (1, 2):
        assert costs[b] == np.inf and not gx[b].any() and not gy[b].any()


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_nan_and_inf_isolation(storage, topo):
    """A NaN or +inf factor makes its utterance's cost NaN; the other utterances' costs and gradients are bitwise what
    they are without it."""
    N, S, T = 4, 40, 70
    px, py, tl, ul = factors(21, N, S, T, topo)
    ul[1] = max(ul[1], 1)
    base = run_loss(px, py, tl, ul, storage, topo)
    px2, py2 = px.copy(), py.copy()
    px2[1, 0, 0] = np.nan
    py2[2, ul[2], tl[2] - 1] = np.inf
    bad = run_loss(px2, py2, tl, ul, storage, topo)
    assert np.isnan(bad[0][[1, 2]]).all()
    for k in range(3):
        assert np.array_equal(bad[k][[0, 3]], base[k][[0, 3]]), k


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", ["fp32", "fp64"])
def test_log_softmax_factors_match_rnnt_loss(storage, topo):
    """px / py gathered from torch.log_softmax(logits): the costs are rnnt_loss's, and autograd through the gather gives
    rnnt_loss's logit gradient."""
    from warprnnt_pytorch import rnnt_lattice_loss, rnnt_loss
    rng = np.random.default_rng(5)
    N, T, U, V = 4, 30, 9, 40
    logits = torch.tensor(rng.standard_normal((N, T, U, V)), device="cuda", dtype=TORCH[storage])
    labels = torch.tensor(rng.integers(1, V, (N, U - 1)), device="cuda", dtype=torch.int32)
    tl = torch.tensor([30, 25, 12, 30], device="cuda", dtype=torch.int32)
    ul = torch.tensor([8, 3, 0, 8 if topo == "regular" else 6], device="cuda", dtype=torch.int32)
    a = logits.clone().requires_grad_()
    c_ref = rnnt_loss(a, labels, tl, ul, reduction="none", rnnt_type=topo)
    c_ref.sum().backward()
    b = logits.clone().requires_grad_()
    lp = torch.log_softmax(b, -1)
    py = lp[..., 0].transpose(1, 2)
    px = torch.gather(lp[:, :, :U - 1], 3, labels[:, None, :, None].expand(N, T, U - 1, 1))[..., 0].transpose(1, 2)
    c = rnnt_lattice_loss(px, py, tl, ul, "none", rnnt_type=topo)
    c.sum().backward()
    rel = 1e-11 if storage == "fp64" else 1e-5
    assert torch.allclose(c, c_ref, rtol=rel, atol=rel)
    rtol, atol = (1e-9, 1e-12) if storage == "fp64" else (1e-4, 1e-6)
    assert torch.allclose(b.grad, a.grad, rtol=rtol, atol=atol), (b.grad - a.grad).abs().max()


@pytest.mark.parametrize("storage", ["fp32", "fp64"])
@pytest.mark.parametrize("T,U", [(1, 1), (2, 2), (3, 3), (5, 4), (4, 5), (6, 3)])
def test_constrained_recipe(T, U, storage):
    """rnnt_lattice_loss(px + py[:, 1:, :], py, ..., rnnt_type='modified') is k2's constrained transducer."""
    from warprnnt_pytorch import rnnt_lattice_loss
    px, py, _, _ = factors(T * 7 + U, 1, U - 1, T)
    x, y = to_dev(px, py, storage, grad=False)
    c = rnnt_lattice_loss(x + y[:, 1:, :], y, *cuda(np.array([T], np.int32), np.array([U - 1], np.int32)), "none",
                          rnnt_type="modified")
    lpb, lpy = lr.utterance_factors(px[0], py[0], T, U)
    ref = lr.constrained_brute_force(lpb, lpy)
    got = c.item()
    if ref == np.inf:
        assert got == np.inf
    else:
        assert abs(got - ref) <= cost_bar(np.array([ref]), storage, 2 * T)[0], (got, ref)


@pytest.mark.parametrize("topo", TOPOLOGIES)
def test_gradcheck_fp64(topo):
    from warprnnt_pytorch import rnnt_lattice_loss
    px, py, tl, ul = factors(8, 3, 3, 5, topo)
    x, y = to_dev(px, py, "fp64")
    tl_, ul_ = cuda(tl, ul)
    assert torch.autograd.gradcheck(lambda a, b: rnnt_lattice_loss(a, b, tl_, ul_, "none", rnnt_type=topo), (x, y))


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", ["fp32", "fp64", "bf16"])
def test_reductions_and_grad_output(storage, topo):
    px, py, tl, ul = factors(31, 5, 20, 40, topo)
    _, _, _, ux, uy = run_loss(px, py, tl, ul, storage, topo)
    rc, rgx, rgy = lr.loss(ux, uy, tl, ul, MOD[topo])
    nf = n_factors(tl, ul, topo)
    w = np.array([0.0, 2.5, -1.0, 0.0, 0.75])
    c, gx, gy, _, _ = run_loss(px, py, tl, ul, storage, topo,
                               grad_output=torch.tensor(w, device="cuda", dtype=torch.float64 if storage == "fp64"
                                                        else torch.float32))
    assert not gx[[0, 3]].any() and not gy[[0, 3]].any()
    assert_grads(gx, rgx * w[:, None, None], storage, nf, np.ones(5, bool))
    assert_grads(gy, rgy * w[:, None, None], storage, nf, np.ones(5, bool))
    for reduction, scale in (("sum", 1.0), ("mean", 1.0 / 5)):
        c, gx, gy, _, _ = run_loss(px, py, tl, ul, storage, topo, reduction)
        assert c.shape == (1,)
        assert abs(c[0] - rc.sum() * scale) <= cost_bar(np.array([rc.sum() * scale]), storage, nf.sum())[0]
        assert_grads(gx, rgx * scale, storage, nf, np.ones(5, bool))
        assert_grads(gy, rgy * scale, storage, nf, np.ones(5, bool))


def test_module_form_and_needs_input_grad():
    from warprnnt_pytorch import RNNTLatticeLoss, rnnt_lattice_loss
    px, py, tl, ul = factors(4, 3, 6, 10)
    x, y = to_dev(px, py, "fp32")
    tl_, ul_ = cuda(tl, ul)
    m = RNNTLatticeLoss(reduction="sum", rnnt_type="modified")
    assert torch.equal(m(x, y, tl_, ul_), rnnt_lattice_loss(x, y, tl_, ul_, "sum", rnnt_type="modified"))
    y2 = y.detach()
    rnnt_lattice_loss(x, y2, tl_, ul_).backward()
    assert x.grad is not None and y2.grad is None
    # k2's width-T slice of a width-(T+1) px is not contiguous: it is copied
    wide = torch.cat([x.detach(), torch.full_like(x[..., :1], -float("inf"))], -1)
    assert torch.equal(rnnt_lattice_loss(wide[..., :-1], y2, tl_, ul_, "none"),
                       rnnt_lattice_loss(x.detach(), y2, tl_, ul_, "none"))


def test_length_mismatch_is_value_error():
    from warprnnt_pytorch import rnnt_lattice_forced_align, rnnt_lattice_loss
    px, py, tl, ul = factors(4, 3, 6, 10)
    x, y = to_dev(px, py, "fp32")
    for t, u in ((tl - 1, ul), (tl, ul - 1)):
        with pytest.raises(ValueError):
            rnnt_lattice_loss(x, y, *cuda(np.maximum(t, 0), np.maximum(u, 0)))
        with pytest.raises(ValueError):
            rnnt_lattice_forced_align(x, y, *cuda(np.maximum(t, 0), np.maximum(u, 0)))
    with pytest.raises(RuntimeError):
        rnnt_lattice_loss(x, y.cpu(), *cuda(tl, ul))


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_wrappers_write_every_element(storage, topo):
    """NaN-prefilled gradients and scores and sentinel frames through the warp_rnnt wrappers: every element written,
    padding zero."""
    from warprnnt_pytorch import warp_rnnt
    N, S, T = 4, 33, 50
    px, py, tl, ul = factors(13, N, S, T, topo)
    x, y = to_dev(px, py, storage, grad=False)
    tl_, ul_ = cuda(tl, ul)
    costs = torch.full((N,), float("nan"), device="cuda", dtype=warp_rnnt.costs_dtype(y))
    ws = warp_rnnt.gpu_lattice_forward(x, y, tl_, ul_, costs, True, rnnt_type=topo)
    gx = torch.full_like(x, float("nan"))
    gy = torch.full_like(y, float("nan"))
    warp_rnnt.gpu_lattice_backward(gx, gy, tl_, ul_, None, 1.0, ws, rnnt_type=topo)
    frames = torch.full((N, S), -7, dtype=torch.int32, device="cuda")
    scores = torch.full((N,), float("nan"), device="cuda", dtype=warp_rnnt.costs_dtype(y))
    warp_rnnt.gpu_lattice_align(x, y, tl_, ul_, frames, scores, rnnt_type=topo)
    torch.cuda.synchronize()
    assert torch.isfinite(costs).all() and torch.isfinite(scores).all()
    assert torch.isfinite(gx).all() and torch.isfinite(gy).all()
    assert not (frames == -7).any()
    gx, gy = gx.double().cpu().numpy(), gy.double().cpu().numpy()
    for b in range(N):
        assert not gy[b, ul[b] + 1:].any() and not gy[b, :, tl[b]:].any()
        assert not gx[b, ul[b]:].any() and not gx[b, :, tl[b]:].any()
        assert (frames[b, ul[b]:] == -1).all()


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", ["fp32", "fp64"])
def test_backward_reads_only_the_workspace(storage, topo):
    from warprnnt_pytorch import rnnt_lattice_loss
    px, py, tl, ul = factors(17, 3, 30, 40, topo)
    tl_, ul_ = cuda(tl, ul)
    x, y = to_dev(px, py, storage)
    rnnt_lattice_loss(x, y, tl_, ul_).backward()
    ref = (x.grad.clone(), y.grad.clone())
    x.grad = y.grad = None
    c = rnnt_lattice_loss(x, y, tl_, ul_)
    with torch.no_grad():
        x.fill_(float("nan"))
        y.normal_()
    c.backward()
    assert torch.equal(x.grad, ref[0]) and torch.equal(y.grad, ref[1])


# ---- alignment --------------------------------------------------------------------------------------------------------
def run_align(px, py, tl, ul, storage, topo):
    from warprnnt_pytorch import rnnt_lattice_forced_align
    x, y = to_dev(px, py, storage, grad=True)
    frames, scores = rnnt_lattice_forced_align(x, y, *cuda(tl, ul), rnnt_type=topo)
    torch.cuda.synchronize()
    assert scores.grad_fn is None and frames.dtype == torch.int32
    assert scores.dtype == (torch.float64 if storage == "fp64" else torch.float32)
    f = lambda t: t.detach().double().cpu().numpy()   # noqa: E731
    return f(scores), frames.cpu().numpy(), f(x), f(y)


def assert_alignment(scores, frames, ux, uy, tl, ul, storage, topo):
    """§12's bars against align_reference.align_factors on the stored factors."""
    mod = MOD[topo]
    s_ref, _ = lr.align(ux, uy, tl, ul, mod)
    assert np.array_equal(np.isnan(scores), np.isnan(s_ref)) and np.array_equal(np.isinf(scores), np.isinf(s_ref))
    fin = np.isfinite(s_ref)
    assert (frames[~fin] == -1).all()
    nf = n_factors(tl, ul, topo)
    assert (np.abs(scores[fin] - s_ref[fin]) <= cost_bar(s_ref[fin], storage, nf[fin])).all(), (scores, s_ref)
    Tb, Ub = lr.extents(tl, ul, ux.shape[2], ux.shape[1])
    for b in np.flatnonzero(fin):
        lpb, lpy = lr.utterance_factors(ux[b], uy[b], Tb[b], Ub[b])
        f = frames[b, :Ub[b] - 1]
        assert ar.valid_alignment(f, Tb[b], Ub[b], mod), (b, f)
        assert (frames[b, Ub[b] - 1:] == -1).all()
        resc = ar.rescore_factors(f, lpb, lpy, mod)
        assert abs(resc - s_ref[b]) <= cost_bar(np.array([s_ref[b]]), storage, nf[b])[0], (b, resc, s_ref[b])


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", ["U1", "U2", "U21", "U33", "U65", "U301", "T1"])
def test_align_against_reference(shape, storage, topo):
    px, py, tl, ul = factors(seed(shape, topo) + 500, *SHAPES[shape], topo=topo)
    scores, frames, ux, uy = run_align(px, py, tl, ul, storage, topo)
    assert_alignment(scores, frames, ux, uy, tl, ul, storage, topo)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_align_planted_paths_exact(storage, topo):
    """+10 on every factor of a random alignment: it is the best path by a wide margin and comes back exactly."""
    N, S, T = 3, 40, 90
    px, py, tl, ul = factors(41, N, S, T, topo)
    rng = np.random.default_rng(42)
    planted = np.full((N, S), -1)
    for b in range(N):
        U = ul[b] + 1
        f = ar.random_alignment(rng, tl[b], U, MOD[topo])
        planted[b, :U - 1] = f
        u = 0
        for t in range(tl[b]):
            if MOD[topo]:
                if u < U - 1 and f[u] == t:
                    px[b, u, t] += 10.0
                    u += 1
                else:
                    py[b, u, t] += 10.0
            else:
                while u < U - 1 and f[u] == t:
                    px[b, u, t] += 10.0
                    u += 1
                py[b, u, t] += 10.0
    scores, frames, ux, uy = run_align(px, py, tl, ul, storage, topo)
    np.testing.assert_array_equal(frames, planted)
    assert_alignment(scores, frames, ux, uy, tl, ul, storage, topo)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_align_uniform_factors_closed_form(storage, topo):
    """Every factor -1/2 (exact in every storage type): every tie is exact, so regular emits every label at frame 0
    and modified label j at frame j; the score is the number of factors times -1/2."""
    N, S, T = 3, 20, 30
    tl = np.array([30, 25, 20], np.int32)
    ul = np.array([20, 7, 0], np.int32)
    px = np.full((N, S, T), -0.5)
    py = np.full((N, S + 1, T), -0.5)
    scores, frames, _, _ = run_align(px, py, tl, ul, storage, topo)
    for b in range(N):
        want = np.arange(ul[b]) if topo == "modified" else np.zeros(ul[b])
        np.testing.assert_array_equal(frames[b, :ul[b]], want)
        nf = n_factors(tl[b], ul[b], topo)
        assert abs(scores[b] + 0.5 * nf) <= cost_bar(np.array([0.5 * nf]), storage, nf)[0]


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_align_no_path_and_nan(storage, topo):
    N, S, T = 4, 10, 12
    px, py, tl, ul = factors(51, N, S, T, topo)
    ul[2] = max(ul[2], 1)
    base_s, base_f, _, _ = run_align(px, py, tl, ul, storage, topo)
    py[1] = -np.inf
    px[2, 0, 0] = np.nan
    py[3, 0, 0] = np.inf
    scores, frames, ux, uy = run_align(px, py, tl, ul, storage, topo)
    assert scores[1] == -np.inf and np.isnan(scores[2]) and np.isnan(scores[3])
    assert (frames[1:] == -1).all()
    assert scores[0] == base_s[0] and np.array_equal(frames[0], base_f[0])


# ---- streams, graphs, launch counts ------------------------------------------------------------------------------
def test_stream_graph_capture_and_launch_counts():
    from warprnnt_pytorch import rnnt_lattice_forced_align, warp_rnnt
    N, S, T = 3, 64, 80
    px, py, tl, ul = factors(61, N, S, T)
    x, y = to_dev(px, py, "fp32", grad=False)
    tl_, ul_ = cuda(tl, ul)
    costs = torch.empty(N, device="cuda")
    ws = warp_rnnt.gpu_lattice_forward(x, y, tl_, ul_, costs, True)
    assert warp_rnnt.last_launch_count() == 2
    gx, gy = torch.empty_like(x), torch.empty_like(y)
    warp_rnnt.gpu_lattice_backward(gx, gy, tl_, ul_, None, 1.0, ws)
    assert warp_rnnt.last_launch_count() == 1
    f0, s0 = rnnt_lattice_forced_align(x, y, tl_, ul_)
    assert warp_rnnt.last_launch_count() == 2

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c1 = torch.empty(N, device="cuda")
        ws1 = warp_rnnt.gpu_lattice_forward(x, y, tl_, ul_, c1, True)
        gx1, gy1 = torch.empty_like(x), torch.empty_like(y)
        warp_rnnt.gpu_lattice_backward(gx1, gy1, tl_, ul_, None, 1.0, ws1)
        f1, s1 = rnnt_lattice_forced_align(x, y, tl_, ul_)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(c1, costs) and torch.equal(gx1, gx) and torch.equal(gy1, gy)
    assert torch.equal(f1, f0) and torch.equal(s1, s0)

    xin, yin = torch.zeros_like(x), torch.zeros_like(y)
    c2 = torch.empty(N, device="cuda")
    gx2, gy2 = torch.empty_like(x), torch.empty_like(y)
    frames = torch.empty((N, S), dtype=torch.int32, device="cuda")
    scores = torch.empty(N, device="cuda")
    ws2 = torch.empty(warp_rnnt.lattice_workspace_size(T, S + 1, N), dtype=torch.uint8, device="cuda")
    ws3 = torch.empty_like(ws2)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        warp_rnnt.gpu_lattice_forward(xin, yin, tl_, ul_, c2, True, ws2)   # warm-up before capture
        side.synchronize()
        with torch.cuda.graph(g, stream=side):
            warp_rnnt.gpu_lattice_forward(xin, yin, tl_, ul_, c2, True, ws2)
            warp_rnnt.gpu_lattice_backward(gx2, gy2, tl_, ul_, None, 1.0, ws2)
            warp_rnnt.gpu_lattice_align(xin, yin, tl_, ul_, frames, scores, ws3)
    xin.copy_(x)
    yin.copy_(y)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(c2, costs) and torch.equal(gx2, gx) and torch.equal(gy2, gy)
    assert torch.equal(frames, f0) and torch.equal(scores, s0)


# ---- ring depth of the multi-warp wavefront (the hook is read once per process) -----------------------------------
CHILD = r"""
import sys, numpy as np, torch
sys.path[:0] = sys.argv[2:]
import test_gpu_lattice as t
from warprnnt_pytorch import warp_rnnt
out = {}
for topo in t.TOPOLOGIES:
    px, py, tl, ul = t.factors(77, 2, 300, 400, topo)
    c, gx, gy, _, _ = t.run_loss(px, py, tl, ul, "fp32", topo)
    out[topo + ".c"], out[topo + ".gx"], out[topo + ".gy"] = c, gx, gy
np.savez(sys.argv[1], depth=warp_rnnt.lib().rnnt_b200_debug_policy(4, 301, 0), **out)
"""


def test_ring_depth_hook(tmp_path):
    """RNNT_B200_LAT_RING = 8, 16, 32 at maxU 301, one process each: bitwise the default (the depth changes when the
    factors arrive, not the arithmetic), and the default against the reference."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("RNNT_B200_")}
    paths = {}
    for ring in ("default", "8", "16", "32"):
        e = dict(env)
        if ring != "default":
            e["RNNT_B200_LAT_RING"] = ring
        paths[ring] = str(tmp_path / ("ring_%s.npz" % ring))
        r = subprocess.run([sys.executable, "-c", CHILD, paths[ring], HERE, os.path.dirname(HERE),
                            os.path.join(os.path.dirname(HERE), "warp-transducer_b200")],
                           env=e, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = {k: np.load(p) for k, p in paths.items()}
    assert [int(res[k]["depth"]) for k in ("default", "8", "16", "32")] == [8, 8, 16, 32]
    for k in ("8", "16", "32"):
        for name in set(res["default"].files) - {"depth"}:
            assert np.array_equal(res[k][name], res["default"][name], equal_nan=True), (k, name)
    for topo in TOPOLOGIES:
        px, py, tl, ul = factors(77, 2, 300, 400, topo)
        ux = torch.tensor(px).float().double().numpy()
        uy = torch.tensor(py).float().double().numpy()
        rc, rgx, rgy = lr.loss(ux, uy, tl, ul, MOD[topo])
        nf = n_factors(tl, ul, topo)
        d = res["default"]
        assert_costs(d[topo + ".c"], rc, "fp32", nf)
        assert_grads(d[topo + ".gx"], rgx, "fp32", nf, np.ones(2, bool))
        assert_grads(d[topo + ".gy"], rgy, "fp32", nf, np.ones(2, bool))
    print(json.dumps({k: int(res[k]["depth"]) for k in res}))
