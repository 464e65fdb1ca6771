"""Forced alignment (DESIGN.md §12) on the GPU against the fp64 reference (tests/align_reference.py).

Bars: scores within §6's cost bar of the fp64 best score, 1e-5 relative (fp64 storage: 1e-11), plus 2^-22 per factor
of the path for the fp32 factors: pass 1 writes each factor as m 2^k with m from ex2.approx (2 ulp), so a path of
T_b + U_b - 1 factors carries that much absolute error in its log-probability whatever the score; it decides the bar
only near score 0 (planted paths).  16-bit storage is compared with the reference on the rounded logits.  The frames
must form a valid alignment whose fp64 rescore lies within the same bar of the best score (robust to near-ties), and
come back exactly where the best path is unique by a wide margin (planted paths) or fixed by the tie rule (uniform
logits)."""
import numpy as np
import pytest
import torch

import align_reference as ar
import pruned_reference as pr
from test_gpu_delay_penalty import STORAGES, TORCH, cuda, make

pytestmark = pytest.mark.gpu

TOPOLOGIES = ["regular", "modified"]
# (N, T, U, V): the pass-1 family each shape reaches for fp32 (16-bit rows are half as long, and never use the chunk
# kernels) and the Viterbi CTA: ceil(U / 32) warps, the decision words of u = 31/32 and 63/64 included
SHAPES = {
    "chunk": (4, 12, 6, 28),              # rows <= 512 B: rowstats_chunk_kernel; one warp
    "tile": (3, 10, 5, 500),              # register tiles
    "row": (2, 6, 4, 1500),               # one CTA per row
    "U33": (3, 40, 33, 20),               # two warps, the last with one column
    "U40": (3, 45, 40, 20),
    "U64": (2, 70, 64, 12),               # two full warps
    "U65": (2, 70, 65, 20),               # three warps
    "U301": (2, 310, 301, 8),             # ten warps
    "T1500": (2, 1500, 301, 8),           # a long backtrace (C4's extents)
}
RUN = {"regular": False, "modified": True}


def bar(ref, storage, factors=0):
    if storage == "fp64":
        return 1e-11 * np.maximum(np.abs(ref), 1.0)
    return 1e-5 * np.maximum(np.abs(ref), 1.0) + factors * 2.0 ** -22


def n_factors(tl, ul, topo):
    return tl if topo == "modified" else tl + ul


def mixed(seed, N, T, U, V, topo):
    """make(); modified: T_b >= U_b - 1 except for one utterance without a path (when N > 2)."""
    acts, labels, tl, ul = make(seed, N, T, U, V)
    if topo == "modified":
        ul[1:] = np.minimum(ul[1:], tl[1:])
        if N > 2:
            tl[N - 1] = max(1, min(T, U - 2) // 2)
            ul[N - 1] = min(U - 1, tl[N - 1] + 1)
    return acts, labels, tl, ul


def run_align(acts_np, labels, tl, ul, storage, topo, ranges=None):
    """(scores, frames, logits as stored in float64) through the public functions."""
    from warprnnt_pytorch import pruned_rnnt_forced_align, rnnt_forced_align
    x = torch.tensor(acts_np, device="cuda").to(TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    if ranges is None:
        frames, scores = rnnt_forced_align(x, lab, tl_, ul_, rnnt_type=topo)
    else:
        frames, scores = pruned_rnnt_forced_align(x, lab, tl_, ul_, cuda(ranges)[0], rnnt_type=topo)
    torch.cuda.synchronize()
    assert frames.dtype == torch.int32 and scores.dtype == (torch.float64 if storage == "fp64" else torch.float32)
    return scores.double().cpu().numpy(), frames.cpu().numpy(), x.double().cpu().numpy()


def assert_alignment(scores, frames, used, labels, tl, ul, storage, topo, ranges=None):
    mod = RUN[topo]
    s_ref, f_ref = ar.align(used, labels, tl, ul, ranges, modified=mod)
    fin = np.isfinite(s_ref)
    assert np.array_equal(np.isfinite(scores), fin), (scores, s_ref)
    assert np.array_equal(np.isnan(scores), np.isnan(s_ref))
    assert (scores[np.isinf(s_ref)] == -np.inf).all()
    assert (frames[~fin] == -1).all()
    nf = n_factors(tl, ul, topo)
    err = np.abs(scores[fin] - s_ref[fin])
    assert (err <= bar(s_ref[fin], storage, nf[fin])).all(), (err / bar(s_ref[fin], storage, nf[fin])).max()
    rescored = ar.rescore(frames, used, labels, tl, ul, ranges, modified=mod)
    for b in np.nonzero(fin)[0]:
        U_b = int(ul[b]) + 1
        assert ar.valid_alignment(frames[b], int(tl[b]), U_b, mod), (b, frames[b])
        assert (frames[b, U_b - 1:] == -1).all()
        assert abs(rescored[b] - s_ref[b]) <= bar(s_ref[b], storage, nf[b]), (b, rescored[b], s_ref[b])
    return s_ref, f_ref


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_against_reference(shape, storage, topo):
    N, T, U, V = SHAPES[shape]
    acts, labels, tl, ul = mixed(1, N, T, U, V, topo)
    scores, frames, used = run_align(acts, labels, tl, ul, storage, topo)
    assert_alignment(scores, frames, used, labels, tl, ul, storage, topo)


def planted(seed, N, T, U, V, topo):
    rng = np.random.default_rng(seed)
    acts, labels, tl, ul = mixed(seed, N, T, U, V, topo)
    want = np.full((N, U - 1), -1, np.int64)
    for b in range(N):
        f = ar.random_alignment(rng, int(tl[b]), int(ul[b]) + 1, RUN[topo])
        if f is None:
            continue
        want[b, :ul[b]] = f
        ar.plant(rng, acts[b], labels[b], f, int(tl[b]), int(ul[b]) + 1, modified=RUN[topo])
    return acts, labels, tl, ul, want


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_planted_path_exact(shape, storage, topo):
    """Random logits with +10 on every transition of a random alignment: that alignment is the unique optimum by a
    wide margin and must come back exactly."""
    N, T, U, V = SHAPES[shape]
    acts, labels, tl, ul, want = planted(2, N, T, U, V, topo)
    scores, frames, used = run_align(acts, labels, tl, ul, storage, topo)
    np.testing.assert_array_equal(frames, want)
    assert_alignment(scores, frames, used, labels, tl, ul, storage, topo)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", ["chunk", "tile", "U33", "U64", "U65", "U301"])
def test_uniform_logits_tie_rule(shape, storage, topo):
    """Every path has the same factors: regular - every label at frame 0, modified - label j at frame j."""
    N, T, U, V = SHAPES[shape]
    _, labels, tl, ul = mixed(3, N, T, U, V, topo)
    acts = np.zeros((N, T, U, V), np.float32)
    scores, frames, used = run_align(acts, labels, tl, ul, storage, topo)
    for b in range(N):
        n = int(ul[b])
        if topo == "modified" and n > tl[b]:
            assert scores[b] == -np.inf and (frames[b] == -1).all()
            continue
        expect = np.arange(n) if topo == "modified" else np.zeros(n)
        np.testing.assert_array_equal(frames[b, :n], expect)
        assert (frames[b, n:] == -1).all()
        factors = n_factors(tl[b], n, topo)
        ref = -factors * np.log(V)
        assert abs(scores[b] - ref) <= bar(ref, storage, factors), (scores[b], ref)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("V", [28, 500])
def test_pruned_random_windows(storage, topo, V):
    """Random monotone windows (for the modified topology some leave no path): the reference on the pruned lattice,
    and every visited cell inside its frame's window."""
    N, T, U, R = 6, 16, 9, 3
    rng = np.random.default_rng(4)
    _, labels, tl, ul = make(4, N, T, U, 2)
    if topo == "modified":
        ul[:] = np.minimum(ul, tl)
    labels = rng.integers(1, V, size=labels.shape).astype(np.int32)
    ranges = pr.random_monotone_ranges(rng, tl, ul, T, R)
    ranges[1, 1:] = R            # frame 1's window starts past frame 0's: no path in either topology
    ul[1] = max(ul[1], R + 1)
    tl[1] = max(tl[1], 2)
    logits = (rng.standard_normal((N, T, R, V)) * 1.5).astype(np.float32)
    scores, frames, used = run_align(logits, labels, tl, ul, storage, topo, ranges)
    s_ref, _ = assert_alignment(scores, frames, used, labels, tl, ul, storage, topo, ranges)
    assert scores[1] == -np.inf and np.isfinite(s_ref).any()
    assert_inside_windows(frames, tl, ul, ranges, R, topo)


def assert_inside_windows(frames, tl, ul, ranges, R, topo):
    for b in range(len(tl)):
        if frames[b, 0] == -1 and ul[b] > 0:
            continue
        f = frames[b, :ul[b]]
        for t in range(int(tl[b])):
            if topo == "modified":
                lo = hi = int(np.searchsorted(f, t, "left"))                     # cell (t, #{j : t_j < t})
            else:
                lo, hi = int(np.searchsorted(f, t, "left")), int(np.searchsorted(f, t, "right"))
            assert ranges[b, t] <= lo and hi <= ranges[b, t] + R - 1, (b, t, lo, hi, ranges[b, t])


@pytest.mark.parametrize("topo", TOPOLOGIES)
def test_pruned_joint_windows(topo):
    """The windows of add_joint_rnnt_loss_with_ranges, and a joiner's logits gathered in them."""
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges, prune_joint_inputs
    N, T, U, V, R = 4, 30, 12, 40, 4
    rng = np.random.default_rng(6)
    _, labels, tl, ul = make(6, N, T, U, V)
    if topo == "modified":
        ul[:] = np.minimum(ul, tl)
    trans = torch.tensor(rng.standard_normal((N, T, V)), dtype=torch.float32, device="cuda")
    pred = torch.tensor(rng.standard_normal((N, U, V)), dtype=torch.float32, device="cuda")
    lab, tl_, ul_ = cuda(labels, tl, ul)
    _, ranges = add_joint_rnnt_loss_with_ranges(trans, pred, lab, tl_, ul_, R, rnnt_type=topo)
    enc, dec = prune_joint_inputs(trans, pred, ranges, R)
    logits = (torch.tanh(enc + dec) * 3.0).contiguous()
    ranges_np = ranges.cpu().numpy()
    scores, frames, used = run_align(logits.cpu().numpy(), labels, tl, ul, "fp32", topo, ranges_np)
    assert_alignment(scores, frames, used, labels, tl, ul, "fp32", topo, ranges_np)
    assert_inside_windows(frames, tl, ul, ranges_np, R, topo)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", ["chunk", "tile", "U40", "U65"])
def test_pruned_full_windows_are_the_dense_alignment_bitwise(shape, storage, topo):
    N, T, U, V = SHAPES[shape]
    acts, labels, tl, ul = mixed(5, N, T, U, V, topo)
    s_d, f_d, _ = run_align(acts, labels, tl, ul, storage, topo)
    s_p, f_p, _ = run_align(acts, labels, tl, ul, storage, topo, np.zeros((N, T), np.int32))
    np.testing.assert_array_equal(f_p, f_d)
    assert np.array_equal(s_p, s_d, equal_nan=True)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_nan_and_minus_inf_logits(storage, topo):
    """A NaN logit: NaN and -1 for that utterance only.  -inf blank logits everywhere: no path, -inf and -1."""
    N, T, U, V = 4, 12, 6, 28
    acts, labels, tl, ul = mixed(6, N, T, U, V, "regular")
    ul[:] = np.minimum(ul, tl)
    ul[1] = ul[2] = 3
    acts[1, 2, 1, 5] = np.nan
    acts[2, :, :, 0] = -np.inf
    scores, frames, used = run_align(acts, labels, tl, ul, storage, topo)
    assert np.isnan(scores[1]) and (frames[1] == -1).all()
    assert scores[2] == -np.inf and (frames[2] == -1).all()
    assert_alignment(scores, frames, used, labels, tl, ul, storage, topo)


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("T,U", [(1, 1), (1, 2), (5, 1), (7, 8), (40, 41), (64, 65), (3, 9), (1, 40)],
                         ids=lambda v: str(v))
def test_edge_extents(T, U, storage, topo):
    """T = 1, no labels (maxU = 1: frames [N, 0]), T_b = U_b - 1 (one modified path: every frame a label), and more
    labels than frames, every utterance full; plus label_len = 0 next to full ones."""
    N, V = 3, 20
    acts, labels, tl, ul = make(2, N, T, U, V)
    tl[:2], ul[:2] = T, U - 1
    ul[2] = 0
    scores, frames, used = run_align(acts, labels, tl, ul, storage, topo)
    assert frames.shape == (N, U - 1)
    assert_alignment(scores, frames, used, labels, tl, ul, storage, topo)
    if topo == "modified" and U - 1 == T:
        np.testing.assert_array_equal(frames[0], np.arange(T))


@pytest.mark.parametrize("topo", TOPOLOGIES)
@pytest.mark.parametrize("storage", STORAGES)
def test_every_output_element_written(storage, topo):
    from warprnnt_pytorch import warp_rnnt
    for shape in ("chunk", "U65"):
        N, T, U, V = SHAPES[shape]
        acts, labels, tl, ul = mixed(7, N, T, U, V, topo)
        x = torch.tensor(acts, device="cuda").to(TORCH[storage])
        lab, tl_, ul_ = cuda(labels, tl, ul)
        frames = torch.full((N, U - 1), -7, dtype=torch.int32, device="cuda")
        scores = torch.full((N,), 12345.0, dtype=warp_rnnt.costs_dtype(x), device="cuda")
        warp_rnnt.gpu_rnnt_align(x, lab, tl_, ul_, frames, scores, 0, rnnt_type=topo)
        assert not (frames == -7).any() and not (scores == 12345.0).any()
        assert (scores.double().cpu().numpy() <= 0.0).all()


@pytest.mark.parametrize("storage", ["fp32", "fp64"])
@pytest.mark.parametrize("topo", TOPOLOGIES)
def test_tunv_equals_ntuv(storage, topo):
    from warprnnt_pytorch import warp_rnnt
    N, T, U, V = SHAPES["U40"]
    acts, labels, tl, ul = mixed(8, N, T, U, V, topo)
    x = torch.tensor(acts, device="cuda").to(TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = []
    for xx, tm in ((x, False), (x.permute(1, 2, 0, 3).contiguous(), True)):
        frames = torch.empty((N, U - 1), dtype=torch.int32, device="cuda")
        scores = torch.empty(N, dtype=x.dtype, device="cuda")
        warp_rnnt.gpu_rnnt_align(xx, lab, tl_, ul_, frames, scores, 0, rnnt_type=topo, time_major=tm)
        out.append((frames.cpu().numpy(), scores.cpu().numpy()))
    np.testing.assert_array_equal(out[0][0], out[1][0])
    assert np.array_equal(out[0][1], out[1][1])


def test_stream_graph_capture_and_launch_counts():
    """A non-default stream, capture into a CUDA graph with replay (no host synchronisation inside the call), and
    2 launches for a dense call, 3 for a pruned one."""
    from warprnnt_pytorch import pruned_rnnt_forced_align, rnnt_forced_align, warp_rnnt
    N, T, U, V = SHAPES["U65"]
    acts, labels, tl, ul = mixed(9, N, T, U, V, "regular")
    x = torch.tensor(acts, device="cuda")
    lab, tl_, ul_ = cuda(labels, tl, ul)
    f0, s0 = rnnt_forced_align(x, lab, tl_, ul_)
    assert warp_rnnt.last_launch_count() == 2
    rg = torch.zeros(N, T, dtype=torch.int32, device="cuda")
    f1, s1 = pruned_rnnt_forced_align(x, lab, tl_, ul_, rg)
    assert warp_rnnt.last_launch_count() == 3
    assert torch.equal(f0, f1) and torch.equal(s0, s1)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        f2, s2 = rnnt_forced_align(x, lab, tl_, ul_)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(f0, f2) and torch.equal(s0, s2)

    frames = torch.empty((N, U - 1), dtype=torch.int32, device="cuda")
    scores = torch.empty(N, dtype=torch.float32, device="cuda")
    ws = torch.empty(warp_rnnt.workspace_size(T, U, N), dtype=torch.uint8, device="cuda")
    xin = torch.zeros_like(x)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        warp_rnnt.gpu_rnnt_align(xin, lab, tl_, ul_, frames, scores, 0, ws)   # warm-up (attributes) before capture
        side.synchronize()
        with torch.cuda.graph(g, stream=side):
            warp_rnnt.gpu_rnnt_align(xin, lab, tl_, ul_, frames, scores, 0, ws)
    xin.copy_(x)
    frames.fill_(-7)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(frames, f0) and torch.equal(scores, s0)


def test_no_autograd_graph():
    from warprnnt_pytorch import rnnt_forced_align
    N, T, U, V = SHAPES["chunk"]
    acts, labels, tl, ul = mixed(10, N, T, U, V, "regular")
    x = torch.tensor(acts, device="cuda", requires_grad=True)
    frames, scores = rnnt_forced_align(x, *cuda(labels, tl, ul))
    assert not scores.requires_grad and scores.grad_fn is None and frames.grad_fn is None
