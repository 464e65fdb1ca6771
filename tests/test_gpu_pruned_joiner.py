"""The pruned fused joiner (DESIGN.md §15) on the GPU: bitwise the fused joiner on the full window, against the masked
fp64 reference (tests/pruned_joiner_reference.py) with the fused joiner's per-element bars (tests/test_gpu_joiner.py,
no floor), against pruned_rnnt_loss / pruned_rnnt_forced_align on the fp32 logits torch's joiner forms over
prune_joint_inputs, and for determinism, side streams, CUDA-graph capture and launch counts."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import align_reference as ar
import joiner_reference as jr
import lattice_reference as lr
import pruned_joiner_reference as pjr
import pruned_reference as pr
import test_gpu_joiner as tg

pytestmark = pytest.mark.gpu

DEV = "cuda"
I32_MAX = 2 ** 31 - 1


def simple_ranges(seed, inputs, R):
    """Window starts from the simple loss of random additive-joint projections (add_joint_rnnt_loss_with_ranges)."""
    import warprnnt_pytorch as w
    enc, pred, weight, _, labels, tl, ul = inputs
    N, T, _ = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    g = torch.Generator().manual_seed(seed)
    am = torch.randn(N, T, V, generator=g).to(DEV)
    lm = torch.randn(N, U, V, generator=g).to(DEV)
    labels = labels.clamp(0, V - 1)
    _, ranges = w.add_joint_rnnt_loss_with_ranges(am, lm, labels, tl, ul, max(R, 2))
    return ranges


def adversarial_ranges(seed, inputs, R):
    """Negative, beyond S_b, non-monotone and +-(2^31 - 1) starts mixed with ordinary ones."""
    enc, pred, _, _, _, tl, ul = inputs
    N, T, _ = enc.shape
    U = pred.shape[1]
    rng = np.random.default_rng(seed)
    r = rng.integers(-R, U + 1, (N, T))
    pick = rng.random((N, T))
    r = np.where(pick < 0.08, I32_MAX, r)
    r = np.where((pick >= 0.08) & (pick < 0.16), -I32_MAX, r)
    r = np.where((pick >= 0.16) & (pick < 0.2), -I32_MAX - 1, r)
    return torch.tensor(r, dtype=torch.int32, device=DEV)


def covered(ranges, R, tl, ul, T, U):
    return pjr.covered(ranges, R, tl, ul, T, U)


def incoming(seed, px, py, ranges, R, tl, ul):
    """Random dpx, dpy with NaN on padding and on every cell no valid row covers (neither may be read)."""
    g = torch.Generator().manual_seed(seed)
    dpx = torch.randn(px.shape, generator=g).to(DEV)
    dpy = torch.randn(py.shape, generator=g).to(DEV)
    N, U, T = py.shape
    mx, my = pjr.factor_masks(ranges, R, tl, ul, T, U)
    dpx[~mx] = float('nan')
    dpy[~my] = float('nan')
    return dpx, dpy


def nan_unselected_pred(inputs, ranges, R):
    """NaN in the pred rows of each utterance that no valid row selects (they must not be read)."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    T, U = enc.shape[1], pred.shape[1]
    sel = covered(ranges, R, tl, ul, T, U).any(1)            # [N, U]
    pred = pred.clone()
    pred[~sel] = float('nan')
    return [enc, pred, weight, bias, labels, tl, ul], sel


def run(inputs, ranges, R, blank, activation, chunk_cells=None, seed=0):
    import warprnnt_pytorch as w
    enc, pred, weight, bias, labels, tl, ul = inputs
    leaves = [x.clone().requires_grad_(True) if x is not None else None for x in (enc, pred, weight, bias)]
    px, py = w.pruned_joiner_log_probs(*leaves, labels, tl, ul, ranges, R, blank, activation=activation,
                                       chunk_cells=chunk_cells)
    dpx, dpy = incoming(seed, px, py, ranges, R, tl, ul)
    torch.autograd.backward([px, py], [dpx, dpy])
    grads = [x.grad if x is not None else None for x in leaves]
    return px.detach(), py.detach(), dpx, dpy, grads


def full_check(inputs, ranges, R, blank, activation, chunk_cells=None):
    inputs, sel = nan_unselected_pred(inputs, ranges, R)
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, _ = enc.shape
    U = pred.shape[1]
    px, py, dpx, dpy, grads = run(inputs, ranges, R, blank, activation, chunk_cells)
    cov = covered(ranges, R, tl, ul, T, U)
    h = tg.reference_h(enc, pred, tl, ul, activation).masked_fill(~cov[..., None], 0)
    px_ref, py_ref = pjr.log_probs(h, weight, bias, labels, tl, ul, ranges, R, blank)
    bar, _ = tg.factor_bar(h, weight, bias, px_ref, py_ref)
    tg.check_factors(px, py, px_ref, py_ref, bar)
    gx, gy = pjr.masked_incoming(dpx, dpy, ranges, R, tl, ul)
    dl = jr.dlogits(h, weight, bias, labels, tl, ul, gx, gy, blank)
    err = tg.dl_error(h, weight, bias, dl, gx, gy, tl, ul, bar)
    tg.check_gradients(grads, h, weight, bias, dl, err, activation, tg.n_chunks(N, T, R, chunk_cells))
    de, dp = grads[0], grads[1]
    for i in range(N):
        assert (de[i, tl[i]:] == 0).all() and (dp[i, ul[i] + 1:] == 0).all(), "padding rows of d_enc / d_pred"
    assert (dp[~sel] == 0).all(), "pred rows no valid row selects"
    return px, py, grads


def bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


@pytest.mark.parametrize("chunk_cells", [None, 1, 37, 64, 1000])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_full_window_is_bitwise_the_fused_joiner(chunk_cells, activation):
    import warprnnt_pytorch as w
    N, T, U, H, V = 4, 13, 7, 64, 29 if chunk_cells == 1 else 500
    inputs = tg.make(chunk_cells or 3, N, T, U, H, V, blank=0)
    enc, pred, weight, bias, labels, tl, ul = inputs
    ranges = torch.zeros(N, T, dtype=torch.int32, device=DEV)
    out = []
    for window in (False, True):
        leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
        if window:
            px, py = w.pruned_joiner_log_probs(*leaves, labels, tl, ul, ranges, U, 0, activation=activation,
                                               chunk_cells=chunk_cells)
        else:
            px, py = w.joiner_log_probs(*leaves, labels, tl, ul, 0, activation=activation, chunk_cells=chunk_cells)
        dpx, dpy = tg.incoming(5, px, py, tl, ul)
        torch.autograd.backward([px, py], [dpx, dpy])
        out.append([px.detach(), py.detach()] + [x.grad for x in leaves])
    for name, a, b in zip(("px", "py", "d_enc", "d_pred", "d_weight", "d_bias"), *out):
        assert torch.equal(bits(a), bits(b)), name


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("H", [16, 640, 1024])
@pytest.mark.parametrize("V", [2, 29, 5000, 5001])
def test_against_masked_fp64_reference(activation, H, V):
    blank = 0 if (H + V) % 2 else V - 1
    inputs = tg.make(H * 7 + V, 4, 9, 6, H, V, blank)
    R = 3
    ranges = simple_ranges(H + V, inputs, R) if V % 2 else adversarial_ranges(H + V, inputs, R)
    full_check(inputs, ranges, R, blank, activation)


@pytest.mark.parametrize("kind", ["simple", "adversarial"])
@pytest.mark.parametrize("R", [1, 2, 5, 9])
def test_window_widths(kind, R):
    """R = 1, R < U, R = U (5) and R > U (9)."""
    inputs = tg.make(R * 3 + len(kind), 5, 11, 5, 128, 300, blank=0)
    if kind == "simple" and R > 1:
        ranges = simple_ranges(R, inputs, R)
    else:
        ranges = adversarial_ranges(R, inputs, R)
    full_check(inputs, ranges, R, 0, "tanh")


@pytest.mark.parametrize("chunk_cells", [1, 3, 37, 64, 100, 1000])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_chunk_edges(chunk_cells, activation):
    """Chunk edges inside a window (3: R = 4), inside an utterance (37, 100), at a tile edge (64), one row per
    chunk, and several slabs of the dW contraction (1000 rows: 16 row tiles)."""
    V = 29 if chunk_cells == 1 else 500
    inputs = tg.make(chunk_cells, 4, 70, 9, 64, V, blank=0)
    R = 4
    ranges = simple_ranges(chunk_cells, inputs, R) if chunk_cells % 2 else adversarial_ranges(chunk_cells, inputs, R)
    full_check(inputs, ranges, R, 0, activation, chunk_cells)


def test_edge_utterances_and_labels():
    """T_b = 1 and S_b = 0 (utterance 2), U = 1, no bias, and labels outside the alphabet."""
    inputs = tg.make(9, 4, 7, 5, 64, 100, bias=False)
    full_check(inputs, simple_ranges(1, inputs, 2), 2, 0, "tanh")
    inputs = tg.make(2, 3, 7, 1, 64, 100)
    px, py, _ = full_check(inputs, torch.zeros(3, 7, dtype=torch.int32, device=DEV), 2, 0, "relu")
    assert px.numel() == 0 and py.shape == (3, 1, 7)
    inputs = tg.make(9, 3, 6, 4, 32, 50, nan_pad=False)
    inputs[4][0, 1] = 50 + 7
    inputs[4][1, 0] = -3
    ranges = torch.zeros(3, 6, dtype=torch.int32, device=DEV)
    ranges[0] = 1
    px, _, _, _, _ = run(inputs, ranges, 2, 0, "tanh")
    tl = inputs[5]
    assert torch.isnan(px[0, 1, :tl[0]]).all() and (px[0, 0] == -float('inf')).all()
    assert torch.isnan(px[1, 0, :tl[1]]).all()


@pytest.fixture
def no_tf32():
    """fp32 matmuls without TF32 for the reference logits, restoring the caller's setting afterwards."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def pruned_logits(enc, pred, weight, bias, ranges, R, activation="tanh"):
    """fp32 [N, T, R, V] logits of torch's joiner over prune_joint_inputs, h rounded to bf16 as the kernel does."""
    import warprnnt_pytorch as w
    enc_p, pred_p = w.prune_joint_inputs(enc, pred, ranges, R)
    s = enc_p.float() + pred_p.float()
    hp = (torch.tanh(s) if activation == "tanh" else torch.relu(s)).to(torch.bfloat16)
    return F.linear(hp.float(), weight.float(), bias.float() if bias is not None else None)


def scatter_rows(x, ranges, R, tl, ul, U):
    """[N, T, R, ...] rows to the dense [N, T, U, ...] cells of the valid rows (others zero)."""
    N, T = ranges.shape
    u = ranges.long()[..., None] + torch.arange(R, device=DEV)
    tb = tl.long().clamp(1, T)[:, None, None]
    sb = ul.long().clamp(0, U - 1)[:, None, None]
    valid = (torch.arange(T, device=DEV)[None, :, None] < tb) & (u >= 0) & (u <= sb)
    out = torch.zeros((N, T, U) + x.shape[3:], dtype=x.dtype, device=DEV)
    b, t, r = valid.nonzero(as_tuple=True)
    out[b, t, u[b, t, r]] = x[b, t, r]
    return out


@pytest.mark.parametrize("rnnt_type", ["regular", "modified"])
@pytest.mark.parametrize("reduction", tg.REDUCTIONS)
@pytest.mark.parametrize("delay_penalty", [0.0, 0.25])
def test_loss_against_pruned_rnnt_loss_on_fp32_logits(rnnt_type, reduction, delay_penalty, no_tf32):
    import warprnnt_pytorch as w
    N, T, U, H, V, R = 4, 12, 6, 256, 300, 3
    inputs = tg.make(33, N, T, U, H, V, nan_pad=False)
    enc, pred, weight, bias, labels, tl, ul = inputs
    if rnnt_type == "modified":
        ul = torch.minimum(ul, tl)
        inputs[6] = ul
    ranges = simple_ranges(7, inputs, R)
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    loss = w.pruned_joiner_rnnt_loss(*leaves, labels, tl, ul, ranges, R, 0, reduction, activation="tanh",
                                     rnnt_type=rnnt_type, delay_penalty=delay_penalty)
    go = torch.linspace(0.5, 1.5, N, device=DEV) if reduction == "none" else torch.ones((), device=DEV) * 0.7
    loss.backward(go if reduction == "none" else go.reshape(1))

    logits = pruned_logits(enc, pred, weight, bias, ranges, R).detach().requires_grad_(True)
    ref = w.pruned_rnnt_loss(logits, labels, tl, ul, ranges, 0, reduction, delay_penalty=delay_penalty,
                             rnnt_type=rnnt_type)
    ref.backward(go if reduction == "none" else go.reshape(1))

    cov = covered(ranges, R, tl, ul, T, U)
    h = tg.reference_h(enc, pred, tl, ul, "tanh").masked_fill(~cov[..., None], 0)
    px_ref, py_ref = pjr.log_probs(h, weight, bias, labels, tl, ul, ranges, R)
    bar, _ = tg.factor_bar(h, weight, bias, px_ref, py_ref)
    tb = tl.clamp(1, T).double()
    pen = delay_penalty * ((tb[:, None, None] - 1) / 2 - torch.arange(T, device=DEV, dtype=torch.float64))
    c64, gx, gy = lr.loss((px_ref + pen).cpu().numpy(), py_ref.cpu().numpy(), tl.cpu().numpy(), ul.cpu().numpy(),
                          rnnt_type == "modified")
    scale = go.double().expand(N) * (1.0 / N if reduction == "mean" else 1.0)
    gx = torch.tensor(gx, device=DEV).abs() * scale[:, None, None]
    gy = torch.tensor(gy, device=DEV).abs() * scale[:, None, None]
    n = (tl.double() + ul.double() + 1)
    bmax = float(bar.max())
    cost_bar = 4 * n * bmax + n * 2.0 ** -20 * (1 + torch.tensor(np.abs(c64), device=DEV))
    if reduction != "none":
        cost_bar = cost_bar.sum().reshape(1) / (N if reduction == "mean" else 1)
    same = loss.detach() == ref.detach()     # +inf where the windows leave an utterance no path
    assert (same | ((loss.detach().double() - ref.detach().double()).abs() <= cost_bar)).all(), (loss, ref)

    dl = scatter_rows(logits.grad.double(), ranges, R, tl, ul, U)
    p = torch.softmax(jr.logits(h, weight, bias), -1) * cov[..., None]
    gsum = (gy.permute(0, 2, 1) + F.pad(gx.permute(0, 2, 1), (0, 1)))[..., None]
    onehots = jr.dlogits(h, weight, bias, labels, tl, ul, gx, gy) + 2 * gsum * p
    eps_occ = 3 * float(n.max()) * bmax + 4 * float(n.max()) * 2.0 ** -22
    err = 2.0 ** -8 * dl.abs() + eps_occ * (onehots + gsum * p) + 4 * bar[..., None] * gsum * p
    tg.check_gradients([x.grad for x in leaves], h, weight, bias, dl, err, "tanh", 1)


def test_utterance_without_a_path(no_tf32):
    """Windows that never reach the last label: that utterance costs +inf and its rows get zero gradients; the
    others, on feasible windows, are unaffected."""
    import warprnnt_pytorch as w
    N, T, U, H, V, R = 3, 10, 4, 64, 50, 2
    inputs = tg.make(12, N, T, U, H, V, nan_pad=False)
    enc, pred, weight, bias, labels, tl, ul = inputs
    ul[1] = 3
    rng = np.random.default_rng(12)
    ranges = torch.tensor(pr.random_monotone_ranges(rng, tl.cpu().numpy(), ul.cpu().numpy(), T, R), device=DEV)
    ranges[1] = -1                       # rows u = -1 (padding) and u = 0 only
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    loss = w.pruned_joiner_rnnt_loss(*leaves, labels, tl, ul, ranges, R, 0, "none")
    loss.backward(torch.ones(N, device=DEV))
    ref = w.pruned_rnnt_loss(pruned_logits(enc, pred, weight, bias, ranges, R), labels, tl, ul, ranges, 0, "none")
    assert loss[1] == float('inf') and ref[1] == float('inf')
    assert torch.isfinite(loss[[0, 2]]).all() and torch.isfinite(ref[[0, 2]]).all()
    assert (leaves[0].grad[1] == 0).all() and (leaves[1].grad[1] == 0).all()
    assert (leaves[0].grad[0] != 0).any() and torch.isfinite(leaves[2].grad).all()


@pytest.mark.parametrize("rnnt_type", ["regular", "modified"])
def test_forced_align_composes(rnnt_type, no_tf32):
    import warprnnt_pytorch as w
    N, T, U, H, V, R = 5, 20, 6, 128, 40, 3
    inputs = tg.make(44, N, T, U, H, V, nan_pad=False)
    enc, pred, weight, bias, labels, tl, ul = inputs
    if rnnt_type == "modified":
        ul = torch.minimum(ul, tl)
        inputs[6] = ul
    ranges = simple_ranges(5, inputs, R)
    px, py = w.pruned_joiner_log_probs(enc, pred, weight, bias, labels, tl, ul, ranges, R)
    frames, scores = w.rnnt_lattice_forced_align(px, py, tl, ul, rnnt_type=rnnt_type)
    logits = pruned_logits(enc, pred, weight, bias, ranges, R)
    f_ref, s_ref = w.pruned_rnnt_forced_align(logits, labels, tl, ul, ranges, rnnt_type=rnnt_type)
    cov = covered(ranges, R, tl, ul, T, U)
    h = tg.reference_h(enc, pred, tl, ul, "tanh").masked_fill(~cov[..., None], 0)
    px_ref, py_ref = pjr.log_probs(h, weight, bias, labels, tl, ul, ranges, R)
    bar, _ = tg.factor_bar(h, weight, bias, px_ref, py_ref)
    mod = rnnt_type == "modified"
    for b in range(N):
        Tb, Ub = int(tl[b]), int(ul[b]) + 1
        if not torch.isfinite(s_ref[b]):
            assert scores[b] == s_ref[b] and torch.equal(frames[b], f_ref[b]), b
            continue
        path_bar = float(bar[b].max()) * (Tb + Ub) + (Tb + Ub) * 2.0 ** -20 * (1 + abs(float(s_ref[b])))
        assert abs(float(scores[b]) - float(s_ref[b])) <= path_bar, b
        if not torch.equal(frames[b], f_ref[b]):   # a tie within the bar: both paths must score alike
            lpb, lpy = lr.utterance_factors(px_ref[b].cpu().numpy(), py_ref[b].cpu().numpy(), Tb, Ub)
            s1 = ar.rescore_factors(frames[b].cpu().numpy(), lpb, lpy, mod)
            s2 = ar.rescore_factors(f_ref[b].cpu().numpy(), lpb, lpy, mod)
            assert abs(s1 - s2) <= 2 * path_bar, b


def test_deterministic():
    inputs = tg.make(3, 4, 30, 9, 256, 700)
    ranges = adversarial_ranges(3, inputs, 4)
    a = run(inputs, ranges, 4, 0, "tanh", chunk_cells=200)
    b = run(inputs, ranges, 4, 0, "tanh", chunk_cells=200)
    for x, y in zip([a[0], a[1]] + a[4], [b[0], b[1]] + b[4]):
        assert torch.equal(bits(x), bits(y))


def test_side_stream_and_graph_capture():
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V, R = 3, 16, 6, 128, 200, 3
    inputs = tg.make(8, N, T, U, H, V)
    enc, pred, weight, bias, labels, tl, ul = inputs
    ranges = simple_ranges(8, inputs, R)
    eager = run(inputs, ranges, R, 0, "relu", chunk_cells=100)
    dpx, dpy = eager[2], eager[3]
    win = dict(ranges=ranges, s_range=R)

    def raw(px, py, ge, gp, gw, gb, ws):
        jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "relu", 100, ws, **win)
        jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, dpx, dpy, ge, gp, gw, gb, 0, "relu", 100, ws,
                               **win)

    outs = [torch.empty_like(eager[0]), torch.empty_like(eager[1]), torch.empty_like(enc), torch.empty_like(pred),
            torch.empty_like(weight), torch.empty_like(bias)]
    ws = torch.empty(jn.workspace_size(T, U, N, H, V, 100, s_range=R), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        raw(*outs, ws)
    torch.cuda.current_stream().wait_stream(side)
    expect = [eager[0], eager[1]] + eager[4]
    for x, y in zip(outs, expect):
        assert torch.equal(x, y)

    for o in outs:
        o.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        raw(*outs, ws)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(outs, expect):
        assert torch.equal(x, y)


@pytest.mark.parametrize("chunk_cells", [None, 64, 50])
def test_launch_counts(chunk_cells):
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V, R = 2, 10, 6, 64, 30, 4
    enc, pred, weight, bias, labels, tl, ul = tg.make(4, N, T, U, H, V)
    ranges = torch.zeros(N, T, dtype=torch.int32, device=DEV)
    chunks = tg.n_chunks(N, T, R, chunk_cells)
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "tanh", chunk_cells, ranges=ranges,
                               s_range=R)
    assert jn.last_launch_count() == 1 + 2 * chunks
    g = [torch.empty_like(x) for x in (enc, pred, weight, bias)]
    jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, torch.zeros_like(px), torch.zeros_like(py), *g,
                           0, "tanh", chunk_cells, ws, ranges=ranges, s_range=R)
    assert jn.last_launch_count() == 5 * chunks + 1
    torch.cuda.synchronize()
