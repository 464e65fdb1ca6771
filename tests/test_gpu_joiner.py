"""The fused joiner (DESIGN.md §14) on the GPU against the fp64 reference (tests/joiner_reference.py) built on the
bf16 h torch forms, against rnnt_loss / rnnt_forced_align on the materialised fp32 logits, and for determinism, side
streams, CUDA-graph capture and launch counts.

Bars are derived per element from the accumulation lengths, with no floor (u = 2^-24, the fp32 unit roundoff; the
tensor core's accumulator may truncate, so each MMA step is charged 2u):
- px, py: the logits carry at most 2 (H + 8) u A of error, A = max_v (sum_k |h_k W_vk| + |bias_v|); lse adds that,
  the exponentials' and the per-thread sums' error (V / 8 + 32) u, and 4 u |lse|.
- dlogits carry the bf16 rounding 2^-8 |dl| plus (|dpx| + |dpy|) p_v times the factors' bar.
- dW, dbias, ds, denc, dpred: the dlogit error carried through |operands|, plus 2 u per MMA step of one stage, one u
  per stage, slab and chunk total, over |dl| |operand|, plus the final bf16 rounding 2^-8 |ref|."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import align_reference as ar
import joiner_blocks as jb
import joiner_reference as jr
import lattice_reference as lr

pytestmark = pytest.mark.gpu

U_ = 2.0 ** -24
DEV = "cuda"


def make(seed, N, T, U, H, V, blank=0, bias=True, nan_pad=True, scale=1.0):
    """Inputs with ragged lengths (utterance 0 full, one utterance with T_b = 1 and S_b = 0 when N > 2) and NaN in
    the padded rows of enc and pred."""
    g = torch.Generator().manual_seed(seed)
    enc = (torch.randn(N, T, H, generator=g) * scale).to(torch.bfloat16)
    pred = (torch.randn(N, U, H, generator=g) * scale).to(torch.bfloat16)
    weight = (torch.randn(V, H, generator=g) * (2.0 / H ** 0.5)).to(torch.bfloat16)
    b = torch.randn(V, generator=g).to(torch.bfloat16) if bias else None
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    tl = torch.randint(max(1, T // 2), T + 1, (N,), generator=g, dtype=torch.int32)
    ul = torch.randint(0, U, (N,), generator=g, dtype=torch.int32)
    tl[0], ul[0] = T, U - 1
    if N > 2:
        tl[2], ul[2] = 1, 0
    if nan_pad:
        for i in range(N):
            enc[i, tl[i]:] = float('nan')
            pred[i, ul[i] + 1:] = float('nan')
    return [x.to(DEV) if x is not None else None for x in (enc, pred, weight, b, labels, tl, ul)]


def reference_h(enc, pred, tl, ul, activation):
    h = jr.hidden(enc, pred, activation)
    cell, _ = jr.masks(tl, ul, enc.shape[1], pred.shape[1])
    return h.masked_fill(~cell[..., None], 0)


def factor_bar(h, weight, bias, px_ref, py_ref):
    """Per-cell bar [N, T, U] of px and py, and the reference lse."""
    H, V = weight.shape[1], weight.shape[0]
    A = h.double().abs() @ weight.double().abs().T
    if bias is not None:
        A = A + bias.double().abs()
    z = jr.logits(h, weight, bias)
    lse = torch.logsumexp(z, -1)
    lse = torch.where(torch.isfinite(lse), lse, torch.zeros_like(lse))
    return 2 * (H + 8) * U_ * A.amax(-1) + (V / 8 + 32) * U_ + 4 * U_ * lse.abs(), lse


def check_factors(px, py, px_ref, py_ref, bar):
    bx = bar[:, :, :-1].permute(0, 2, 1)
    by = bar.permute(0, 2, 1)
    for got, ref, b in ((px, px_ref, bx), (py, py_ref, by)):
        ref = ref.to(got.device)
        inf = torch.isinf(ref)
        assert torch.equal(got[inf], ref[inf].float()), "padding must be -inf"
        nan = torch.isnan(ref)
        assert torch.isnan(got[nan]).all()
        ok = ~(inf | nan)
        err = (got[ok].double() - ref[ok]).abs()
        assert (err <= b[ok]).all(), (err.max().item(), (err / b[ok]).max().item())


def gradient_bars(ht, ag, weight, dl, dl_err, chunks, slabs=16):
    """fp64 (d_enc, d_pred, d_weight, d_bias) of dl with ht as dW's operand and ag as ds's factor, and each one's bar
    without the final bf16 rounding 2^-8 |ref|."""
    N, T, U, _ = ht.shape
    V = weight.shape[0]
    ha, wa, dla = ht.double().abs(), weight.double().abs(), dl.abs()
    ds_ref = (dl @ weight.double()) * ag
    ref = (ds_ref.sum(2), ds_ref.sum(1), torch.einsum('ntuv,ntuh->vh', dl, ht.double()), dl.sum((0, 1, 2)))
    g_dw = (32 + N * T * U / 256 + slabs + chunks) * 2 * U_
    g_ds = (32 + V / 256) * 2 * U_
    b_ds = ((dl_err @ wa) + g_ds * (dla @ wa)) * ag
    bars = (b_ds.sum(2) + (U + chunks) * 2 * U_ * ds_ref.abs().sum(2),
            b_ds.sum(1) + (T + chunks) * 2 * U_ * ds_ref.abs().sum(1),
            torch.einsum('ntuv,ntuh->vh', dl_err, ha) + g_dw * torch.einsum('ntuv,ntuh->vh', dla, ha),
            dl_err.sum((0, 1, 2)) + g_dw * dla.sum((0, 1, 2)))
    return ref, bars


def check_gradients(got, h, weight, bias, dl, dl_err, activation, chunks, slabs=16):
    """Each of (d_enc, d_pred, d_weight, d_bias) within its bar of the fp64 contraction of dl."""
    ref, bars = gradient_bars(h, jr.act_grad(h, activation), weight, dl, dl_err, chunks, slabs)
    for name, g, r, b in zip(("d_enc", "d_pred", "d_weight", "d_bias"), got, ref, bars):
        if g is None:
            continue
        err = (g.double() - r).abs()
        lim = b + 2.0 ** -8 * r.abs()
        bad = err > lim
        assert not bad.any(), (name, int(bad.sum()), err.max().item(), (err / lim.clamp_min(1e-300)).max().item())


def dl_error(h, weight, bias, dl, dpx, dpy, tl, ul, bar):
    """Bound on |dl_kernel - dl_ref| per element: the bf16 rounding and the softmax's error through the factors'."""
    N, T, U, _ = h.shape
    p = torch.softmax(jr.logits(h, weight, bias), -1)
    cell, lab = jr.masks(tl, ul, T, U)
    gy = dpy.double().permute(0, 2, 1).abs() * cell
    gx = torch.zeros_like(gy)
    gx[..., :U - 1] = dpx.double().permute(0, 2, 1).abs() * lab
    p = torch.where(cell[..., None], p, torch.zeros_like(p))
    return 2.0 ** -8 * dl.abs() + ((gx + gy) * 2 * bar)[..., None] * p


def incoming(seed, px, py, tl, ul):
    """Random dpx, dpy with NaN on padding (it must not be read)."""
    g = torch.Generator().manual_seed(seed)
    dpx = torch.randn(px.shape, generator=g).to(DEV)
    dpy = torch.randn(py.shape, generator=g).to(DEV)
    N, S1, T = py.shape
    cell, lab = jr.masks(tl, ul, T, S1)
    dpy[~cell.permute(0, 2, 1)] = float('nan')
    dpx[~lab.permute(0, 2, 1)] = float('nan')
    return dpx, dpy


def run(inputs, blank, activation, chunk_cells=None, seed=0):
    import warprnnt_pytorch as w
    enc, pred, weight, bias, labels, tl, ul = inputs
    leaves = [x.clone().requires_grad_(True) if x is not None else None for x in (enc, pred, weight, bias)]
    px, py = w.joiner_log_probs(*leaves, labels, tl, ul, blank, activation=activation, chunk_cells=chunk_cells)
    dpx, dpy = incoming(seed, px, py, tl, ul)
    torch.autograd.backward([px, py], [dpx, dpy])
    grads = [x.grad if x is not None else None for x in leaves]
    return px.detach(), py.detach(), dpx, dpy, grads


def n_chunks(N, T, U, chunk_cells):
    cells = N * T * U
    return 1 if chunk_cells is None else -(-cells // min(chunk_cells, cells))


def full_check(inputs, blank, activation, chunk_cells=None):
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, _ = enc.shape
    U = pred.shape[1]
    px, py, dpx, dpy, grads = run(inputs, blank, activation, chunk_cells)
    h = reference_h(enc, pred, tl, ul, activation)
    px_ref, py_ref = jr.log_probs(h, weight, bias, labels, tl, ul, blank)
    bar, _ = factor_bar(h, weight, bias, px_ref, py_ref)
    check_factors(px, py, px_ref, py_ref, bar)
    dz = lambda x: torch.nan_to_num(x, nan=0.0)   # padding entries are not read
    dl = jr.dlogits(h, weight, bias, labels, tl, ul, dz(dpx), dz(dpy), blank)
    err = dl_error(h, weight, bias, dl, dz(dpx), dz(dpy), tl, ul, bar)
    check_gradients(grads, h, weight, bias, dl, err, activation, n_chunks(N, T, U, chunk_cells))
    de, dp = grads[0], grads[1]
    for i in range(N):
        assert (de[i, tl[i]:] == 0).all() and (dp[i, ul[i] + 1:] == 0).all(), "padding rows of d_enc / d_pred"
    return px, py, grads


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("H", [16, 512, 640, 1024])
@pytest.mark.parametrize("V", [2, 29, 500, 5000, 5001])
def test_against_fp64_reference(activation, H, V):
    blank = 0 if (H + V) % 2 else V - 1
    inputs = make(H * 7 + V, 4, 9, 5, H, V, blank)
    full_check(inputs, blank, activation)


@pytest.mark.parametrize("chunk_cells", [1, 37, 64, 100, 1000])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_chunk_edges(chunk_cells, activation):
    """Chunk edges inside an utterance (37, 100), at a tile edge (64), one cell per chunk, and several slabs of
    the dW contraction (1000 cells: 16 row tiles)."""
    V = 29 if chunk_cells == 1 else 500
    inputs = make(chunk_cells, 4, 13, 7, 64, V, blank=0)
    full_check(inputs, 0, activation, chunk_cells)


def test_many_row_tiles_and_slabs():
    inputs = make(5, 4, 40, 12, 128, 29, blank=3)
    full_check(inputs, 3, "tanh")
    full_check(inputs, 3, "relu", chunk_cells=700)


def test_no_bias_and_single_context():
    full_check(make(1, 3, 7, 4, 64, 100, bias=False), 0, "tanh")
    px, py, grads = full_check(make(2, 3, 7, 1, 64, 100), 0, "tanh")    # U = 1: no labels, px is empty
    assert px.numel() == 0 and py.shape == (3, 1, 7)


def test_label_outside_the_alphabet():
    inputs = make(9, 3, 6, 4, 32, 50, nan_pad=False)
    inputs[4][0, 1] = 50 + 7
    inputs[4][1, 0] = -3
    enc, pred, weight, bias, labels, tl, ul = inputs
    px, py, _, _, _ = run(inputs, 0, "tanh")
    assert torch.isnan(px[0, 1, :tl[0]]).all() and torch.isnan(px[1, 0, :tl[1]]).all()
    h = reference_h(enc, pred, tl, ul, "tanh")
    px_ref, py_ref = jr.log_probs(h, weight, bias, labels, tl, ul)
    bar, _ = factor_bar(h, weight, bias, px_ref, py_ref)
    check_factors(px, py, px_ref, py_ref, bar)


def _plan_h_offset(N, T, U, H, V, chunk):
    """Byte offset of the h scratch in the workspace (rnnt_joiner.cu, plan(); mirrored in joiner_blocks.plan)."""
    p = jb.plan(T, U, N, H, V, chunk)
    return p.h, p.Hp


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_kernel_h_equals_torch_h(activation):
    """The kernel's tanhf and torch's tanh come from different CUDA releases; a one-ulp difference could flip a bf16
    rounding.  Read the kernel's own h (chunk_cells >= the cell count, so the scratch holds every cell)."""
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 4, 50, 20, 1024, 32
    enc, pred, weight, bias, labels, tl, ul = make(21, N, T, U, H, V, scale=1.5)
    cells = N * T * U
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, activation, chunk_cells=cells)
    torch.cuda.synchronize()
    off, Hp = _plan_h_offset(N, T, U, H, V, cells)
    hk = ws[off:off + cells * Hp * 2].view(torch.bfloat16).view(N, U, T, Hp)[..., :H].permute(0, 2, 1, 3)
    href = reference_h(enc, pred, tl, ul, activation)
    flips = int((hk.view(torch.int16) != href.view(torch.int16)).sum())
    assert flips == 0, "%d of %d h elements differ from torch's" % (flips, href.numel())
    assert (ws[off:off + cells * Hp * 2].view(torch.bfloat16).view(cells, Hp)[:, H] == 1).all()


REDUCTIONS = ["none", "sum", "mean"]


@pytest.mark.parametrize("rnnt_type", ["regular", "modified"])
@pytest.mark.parametrize("reduction", REDUCTIONS)
@pytest.mark.parametrize("delay_penalty", [0.0, 0.25])
def test_loss_against_rnnt_loss_on_fp32_logits(rnnt_type, reduction, delay_penalty):
    import warprnnt_pytorch as w
    N, T, U, H, V = 4, 12, 5, 256, 300
    enc, pred, weight, bias, labels, tl, ul = make(33, N, T, U, H, V, nan_pad=False)
    if rnnt_type == "modified":
        ul = torch.minimum(ul, tl)
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    loss = w.joiner_rnnt_loss(*leaves, labels, tl, ul, 0, reduction, activation="tanh", rnnt_type=rnnt_type,
                              delay_penalty=delay_penalty)
    go = torch.linspace(0.5, 1.5, N, device=DEV) if reduction == "none" else torch.ones((), device=DEV) * 0.7
    loss.backward(go if reduction == "none" else go.reshape(1))

    torch.backends.cuda.matmul.allow_tf32 = False
    h = reference_h(enc, pred, tl, ul, "tanh")
    logits = F.linear(h.float(), weight.float(), bias.float()).detach().requires_grad_(True)
    ref = w.rnnt_loss(logits, labels, tl, ul, 0, reduction, delay_penalty=delay_penalty, rnnt_type=rnnt_type)
    ref.backward(go if reduction == "none" else go.reshape(1))

    # fp64 lattice on the fp64 factors: the occupancies that scale each dlogit's error
    px_ref, py_ref = jr.log_probs(h, weight, bias, labels, tl, ul)
    bar, _ = factor_bar(h, weight, bias, px_ref, py_ref)
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
    assert ((loss.detach().double() - ref.detach().double()).abs() <= cost_bar).all(), (loss, ref)

    dl = logits.grad.double()
    p = torch.softmax(jr.logits(h, weight, bias), -1)
    gsum = (gy.permute(0, 2, 1) + F.pad(gx.permute(0, 2, 1), (0, 1)))[..., None]   # |dpx| + |dpy| per cell
    onehots = jr.dlogits(h, weight, bias, labels, tl, ul, gx, gy) + 2 * gsum * p   # |dpy| [blank] + |dpx| [label]
    eps_occ = 3 * float(n.max()) * bmax + 4 * float(n.max()) * 2.0 ** -22
    err = 2.0 ** -8 * dl.abs() + eps_occ * (onehots + gsum * p) + 4 * bar[..., None] * gsum * p
    check_gradients([x.grad for x in leaves], h, weight, bias, dl, err, "tanh", 1)


@pytest.mark.parametrize("rnnt_type", ["regular", "modified"])
def test_forced_align_composes(rnnt_type):
    import warprnnt_pytorch as w
    N, T, U, H, V = 5, 20, 6, 128, 40
    enc, pred, weight, bias, labels, tl, ul = make(44, N, T, U, H, V, nan_pad=False)
    if rnnt_type == "modified":
        ul = torch.minimum(ul, tl)
    px, py = w.joiner_log_probs(enc, pred, weight, bias, labels, tl, ul)
    frames, scores = w.rnnt_lattice_forced_align(px, py, tl, ul, rnnt_type=rnnt_type)
    h = reference_h(enc, pred, tl, ul, "tanh")
    logits = F.linear(h.float(), weight.float(), bias.float())
    f_ref, s_ref = w.rnnt_forced_align(logits, labels, tl, ul, rnnt_type=rnnt_type)
    px_ref, py_ref = jr.log_probs(h, weight, bias, labels, tl, ul)
    bar, _ = factor_bar(h, weight, bias, px_ref, py_ref)
    mod = rnnt_type == "modified"
    for b in range(N):
        Tb, Ub = int(tl[b]), int(ul[b]) + 1
        path_bar = float(bar[b].max()) * (Tb + Ub) + (Tb + Ub) * 2.0 ** -20 * (1 + abs(float(s_ref[b])))
        assert abs(float(scores[b]) - float(s_ref[b])) <= path_bar, b
        if not torch.equal(frames[b], f_ref[b]):   # a tie within the bar: both paths must score alike
            lpb, lpy = lr.utterance_factors(px_ref[b].cpu().numpy(), py_ref[b].cpu().numpy(), Tb, Ub)
            s1 = ar.rescore_factors(frames[b].cpu().numpy(), lpb, lpy, mod)
            s2 = ar.rescore_factors(f_ref[b].cpu().numpy(), lpb, lpy, mod)
            assert abs(s1 - s2) <= 2 * path_bar, b


def test_deterministic():
    inputs = make(3, 4, 30, 9, 256, 700)
    a = run(inputs, 0, "tanh", chunk_cells=200)
    b = run(inputs, 0, "tanh", chunk_cells=200)
    for x, y in zip([a[0], a[1]] + a[4], [b[0], b[1]] + b[4]):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_side_stream_and_graph_capture():
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 3, 16, 6, 128, 200
    enc, pred, weight, bias, labels, tl, ul = make(8, N, T, U, H, V)
    eager = run([enc, pred, weight, bias, labels, tl, ul], 0, "relu", chunk_cells=100)
    dpx, dpy = eager[2], eager[3]

    def raw(px, py, ge, gp, gw, gb, ws):
        jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "relu", 100, ws)
        jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, dpx, dpy, ge, gp, gw, gb, 0, "relu", 100, ws)

    outs = [torch.empty_like(eager[0]), torch.empty_like(eager[1]), torch.empty_like(enc), torch.empty_like(pred),
            torch.empty_like(weight), torch.empty_like(bias)]
    ws = torch.empty(jn.workspace_size(T, U, N, H, V, 100), dtype=torch.uint8, device=DEV)
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
    N, T, U, H, V = 2, 10, 6, 64, 30
    inputs = make(4, N, T, U, H, V)
    enc, pred, weight, bias, labels, tl, ul = inputs
    chunks = n_chunks(N, T, U, chunk_cells)
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "tanh", chunk_cells)
    assert jn.last_launch_count() == 2 * chunks
    g = [torch.empty_like(x) for x in (enc, pred, weight, bias)]
    jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, torch.zeros_like(px), torch.zeros_like(py), *g,
                           0, "tanh", chunk_cells, ws)
    assert jn.last_launch_count() == 5 * chunks + 1
    torch.cuda.synchronize()
