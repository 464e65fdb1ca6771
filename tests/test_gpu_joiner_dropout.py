"""Dropout on the fused and pruned fused joiners' hidden activation (DESIGN.md §16) on the GPU: the kernel's h~ bit
for bit against the reference mask (tests/dropout_reference.py), the factors and gradients against the fp64 reference
on h~ with the fused joiner's per-element bars (tests/test_gpu_joiner.py, no floor), p = 0 as the plain entries, the
pruned identities, rnnt_loss / pruned_rnnt_loss on the fp32 logits of torch's joiner with the same mask, the seed's
RNG behaviour, side streams, CUDA graphs and launch counts.

The bars are test_gpu_joiner.py's with h~ for h in the logits and dW, and act'(s) keep scale for act'(s) in ds."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_reference as dr
import joiner_blocks as jb
import joiner_reference as jr
import lattice_reference as lr
import pruned_joiner_reference as pjr
import test_gpu_joiner as tg
import test_gpu_pruned_joiner as tp

pytestmark = pytest.mark.gpu

U_ = 2.0 ** -24
DEV = "cuda"


def seed_tensor(s):
    return torch.tensor([s], dtype=torch.int64, device=DEV)


def bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


def reference(inputs, activation, p, seed, window=None):
    """(h, mask, h~): torch's bf16 h (zero off the valid cells; pruned: off the covered cells), the keep mask of the
    padded grid and h~."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, H = enc.shape
    U = pred.shape[1]
    h = tg.reference_h(enc, pred, tl, ul, activation)
    if window is not None:
        h = h.masked_fill(~pjr.covered(window[0], window[1], tl, ul, T, U)[..., None], 0)
    mask = dr.keep_mask(seed, N, T, U, H, p).to(DEV)
    return h, mask, dr.dropped_hidden(h, mask, p)


def check_gradients(got, ht, ag, weight, dl, dl_err, chunks, slabs=16):
    """test_gpu_joiner.check_gradients with h~ as dW's operand and ag = act' keep scale as ds's factor."""
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
    for name, g, r, b in zip(("d_enc", "d_pred", "d_weight", "d_bias"), got, ref, bars):
        if g is None:
            continue
        err = (g.double() - r).abs()
        lim = b + 2.0 ** -8 * r.abs()
        bad = err > lim
        assert not bad.any(), (name, int(bad.sum()), err.max().item(), (err / lim.clamp_min(1e-300)).max().item())


def run(inputs, blank, activation, p, seed, chunk_cells=None, window=None, grad_seed=0):
    import warprnnt_pytorch as w
    enc, pred, weight, bias, labels, tl, ul = inputs
    leaves = [x.clone().requires_grad_(True) if x is not None else None for x in (enc, pred, weight, bias)]
    kw = dict(activation=activation, chunk_cells=chunk_cells, dropout=p,
              dropout_seed=seed_tensor(seed) if seed is not None else None)
    if window is None:
        px, py = w.joiner_log_probs(*leaves, labels, tl, ul, blank, **kw)
        dpx, dpy = tg.incoming(grad_seed, px, py, tl, ul)
    else:
        px, py = w.pruned_joiner_log_probs(*leaves, labels, tl, ul, *window, blank, **kw)
        dpx, dpy = tp.incoming(grad_seed, px, py, *window, tl, ul)
    torch.autograd.backward([px, py], [dpx, dpy])
    return px.detach(), py.detach(), dpx, dpy, [x.grad if x is not None else None for x in leaves]


def full_check(inputs, blank, activation, p, seed, chunk_cells=None, window=None):
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, _ = enc.shape
    U = pred.shape[1]
    px, py, dpx, dpy, grads = run(inputs, blank, activation, p, seed, chunk_cells, window)
    h, mask, ht = reference(inputs, activation, p, seed, window)
    if window is None:
        px_ref, py_ref = dr.log_probs(ht, weight, bias, labels, tl, ul, blank)
        gx, gy = torch.nan_to_num(dpx, nan=0.0), torch.nan_to_num(dpy, nan=0.0)   # padding is not read
    else:
        px_ref, py_ref = dr.pruned_log_probs(ht, weight, bias, labels, tl, ul, *window, blank)
        gx, gy = pjr.masked_incoming(dpx, dpy, *window, tl, ul)
    bar, _ = tg.factor_bar(ht, weight, bias, px_ref, py_ref)
    tg.check_factors(px, py, px_ref, py_ref, bar)
    dl = jr.dlogits(ht, weight, bias, labels, tl, ul, gx, gy, blank)
    err = tg.dl_error(ht, weight, bias, dl, gx, gy, tl, ul, bar)
    rows = window[1] if window is not None else U
    check_gradients(grads, ht, dr.act_grad(h, mask, p, activation), weight, dl, err,
                    tg.n_chunks(N, T, rows, chunk_cells))
    for i in range(N):
        assert (grads[0][i, tl[i]:] == 0).all() and (grads[1][i, ul[i] + 1:] == 0).all()
    return px, py, grads


# 1. the kernel's h~ is the reference's bit for bit

def _h_offset(N, T, U, rows_per_frame, H, V, chunk):
    """Byte offset of the h scratch in the workspace (rnnt_joiner.cu, plan(); mirrored in joiner_blocks.plan), and
    Hp."""
    p = jb.plan(T, U, N, H, V, chunk, rows_per_frame)
    return p.h, p.Hp


@pytest.mark.parametrize("pruned", [False, True])
@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
@pytest.mark.parametrize("H", [16, 640, 1024])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_kernel_h_is_the_reference_h_tilde(activation, H, p, pruned):
    """The scratch after a forward holds the last chunk's rows: with chunk_cells >= the row count every row, with a
    smaller chunk (a chunk edge inside an utterance) the last chunk's."""
    import warprnnt_pytorch.joiner as jn
    N, T, U, V, R = 3, 11, 5, 32, 3
    seed = H * 1000 + int(p * 10) + (2 ** 40 if pruned else 0)
    inputs = tg.make(H + int(p * 10), N, T, U, H, V, scale=1.5)
    enc, pred, weight, bias, labels, tl, ul = inputs
    window = (tp.adversarial_ranges(H, inputs, R), R) if pruned else None
    rpf = R if pruned else U
    rows = N * T * rpf
    h, mask, ht = reference(inputs, activation, p, seed, window)
    if pruned:   # the rows (b, r, t) of the windows: the covered cell's h~, 0 on padding rows
        ranges = window[0].long()
        u = ranges[:, None, :] + torch.arange(R, device=DEV)[None, :, None]            # [N, R, T]
        t = torch.arange(T, device=DEV)[None, None, :].expand(N, R, T)
        b = torch.arange(N, device=DEV)[:, None, None].expand(N, R, T)
        valid = (t < tl.long().clamp(1, T)[:, None, None]) & (u >= 0) & (u <= ul.long().clamp(0, U - 1)[:, None, None])
        expect = torch.zeros(N, R, T, H, dtype=torch.bfloat16, device=DEV)
        expect[valid] = ht[b[valid], t[valid], u[valid]]
        expect = expect.reshape(rows, H)
    else:
        expect = ht.permute(0, 2, 1, 3).reshape(rows, H)
    for chunk in (rows, 37):
        px = torch.empty(N, U - 1, T, device=DEV)
        py = torch.empty(N, U, T, device=DEV)
        ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, activation, chunk,
                                   ranges=window[0] if pruned else None, s_range=R if pruned else None,
                                   dropout=p, seed=seed_tensor(seed))
        torch.cuda.synchronize()
        off, Hp = _h_offset(N, T, U, rpf, H, V, chunk)
        c0 = (rows - 1) // chunk * chunk
        got = ws[off:off + (rows - c0) * Hp * 2].view(torch.bfloat16).view(rows - c0, Hp)
        flips = int((got[:, :H].view(torch.int16) != expect[c0:].view(torch.int16)).sum())
        assert flips == 0, "%d of %d h~ elements differ (chunk %d)" % (flips, expect[c0:].numel(), chunk)
        assert (got[:, H] == 1).all(), "the bias column is never dropped"
    kept = mask[h != 0].float().mean().item()
    assert abs(kept - (1 - p)) < 0.1


# 2. factors and gradients against the fp64 reference on h~

@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("V", [29, 5000, 5001])
@pytest.mark.parametrize("pruned", [False, True])
def test_against_fp64_reference(activation, V, pruned):
    blank = 0 if V % 2 else V - 1
    inputs = tg.make(V + 3, 4, 9, 5, 128, V, blank)
    window = (tp.simple_ranges(V, inputs, 3) if V % 2 else tp.adversarial_ranges(V, inputs, 3), 3) if pruned \
        else None
    full_check(inputs, blank, activation, 0.2, V * 7 + 1, window=window)


@pytest.mark.parametrize("chunk_cells", [1, 37, 1000])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_chunk_edges_and_slabs(chunk_cells, activation):
    """One cell per chunk, chunk edges inside an utterance, and several dW slabs (1000 cells: 16 row tiles)."""
    V = 29 if chunk_cells == 1 else 500
    inputs = tg.make(chunk_cells, 4, 13, 7, 64, V, blank=0)
    full_check(inputs, 0, activation, 0.5 if chunk_cells == 37 else 0.1, chunk_cells, chunk_cells)
    if chunk_cells != 1:
        full_check(inputs, 0, activation, 0.2, chunk_cells + 1, chunk_cells, (tp.simple_ranges(3, inputs, 4), 4))


def test_edge_utterances():
    """T_b = 1 and S_b = 0 (utterance 2), U = 1, no bias."""
    full_check(tg.make(1, 3, 7, 4, 64, 100, bias=False), 0, "tanh", 0.2, 11)
    px, py, _ = full_check(tg.make(2, 3, 7, 1, 64, 100), 0, "relu", 0.2, 12)
    assert px.numel() == 0 and py.shape == (3, 1, 7)


# 3. p = 0 is the plain path

def _always_drop_entries(jn):
    def entry(name, dropout, seed):
        return getattr(jn._lib, name + "_drop"), [jn.rnntJoinerDropout(dropout, _ptr(seed))]
    return entry


def _ptr(seed):
    return seed.data_ptr() if seed is not None else None


@pytest.mark.parametrize("pruned", [False, True])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_p0_drop_entries_are_bitwise_the_plain_entries(activation, pruned, monkeypatch):
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 3, 9, 5, 128, 300
    inputs = tg.make(5, N, T, U, H, V)
    window = (tp.simple_ranges(5, inputs, 3), 3) if pruned else None
    plain = run(inputs, 0, activation, 0.0, None, 100, window)
    with monkeypatch.context() as m:
        m.setattr(jn, "_drop", _always_drop_entries(jn))
        for seed in (None, 7):   # the seed is not read at p = 0
            drop = run(inputs, 0, activation, 0.0, seed, 100, window)
            for a, b in zip([plain[0], plain[1]] + plain[4], [drop[0], drop[1]] + drop[4]):
                assert torch.equal(bits(a), bits(b))


def test_python_dropout_zero_is_the_plain_call():
    import warprnnt_pytorch as w
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 2, 10, 6, 64, 30
    enc, pred, weight, bias, labels, tl, ul = tg.make(4, N, T, U, H, V)
    a = w.joiner_log_probs(enc, pred, weight, bias, labels, tl, ul, chunk_cells=50)
    b = w.joiner_log_probs(enc, pred, weight, bias, labels, tl, ul, chunk_cells=50, dropout=0.0)
    assert jn.last_launch_count() == 2 * tg.n_chunks(N, T, U, 50)
    for x, y in zip(a, b):
        assert torch.equal(bits(x), bits(y))


# 4. the pruned identities with dropout on

@pytest.mark.parametrize("chunk_cells", [None, 37])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_full_window_is_bitwise_the_dense_call(chunk_cells, activation):
    N, T, U, H, V = 4, 13, 7, 64, 500
    inputs = tg.make(17, N, T, U, H, V)
    zero = torch.zeros(N, T, dtype=torch.int32, device=DEV)
    a = run(inputs, 0, activation, 0.2, 99, chunk_cells)
    b = run(inputs, 0, activation, 0.2, 99, chunk_cells, (zero, U))
    for name, x, y in zip(("px", "py", "d_enc", "d_pred", "d_weight", "d_bias"), [a[0], a[1]] + a[4],
                          [b[0], b[1]] + b[4]):
        assert torch.equal(bits(x), bits(y)), name


# 5. against rnnt_loss / pruned_rnnt_loss on the fp32 logits of torch's joiner with the same mask

@pytest.mark.parametrize("pruned", [False, True])
@pytest.mark.parametrize("rnnt_type", ["regular", "modified"])
@pytest.mark.parametrize("reduction", tg.REDUCTIONS)
@pytest.mark.parametrize("delay_penalty", [0.0, 0.25])
def test_loss_against_eager_dropout(pruned, rnnt_type, reduction, delay_penalty, no_tf32):
    import warprnnt_pytorch as w
    N, T, U, H, V, R, p, seed = 4, 12, 6, 256, 300, 3, 0.2, 2024
    inputs = tg.make(33, N, T, U, H, V, nan_pad=False)
    enc, pred, weight, bias, labels, tl, ul = inputs
    if rnnt_type == "modified":
        ul = torch.minimum(ul, tl)
        inputs[6] = ul
    ranges = tp.simple_ranges(7, inputs, R) if pruned else None
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    kw = dict(activation="tanh", rnnt_type=rnnt_type, delay_penalty=delay_penalty, dropout=p,
              dropout_seed=seed_tensor(seed))
    if pruned:
        loss = w.pruned_joiner_rnnt_loss(*leaves, labels, tl, ul, ranges, R, 0, reduction, **kw)
    else:
        loss = w.joiner_rnnt_loss(*leaves, labels, tl, ul, 0, reduction, **kw)
    go = torch.linspace(0.5, 1.5, N, device=DEV) if reduction == "none" else torch.ones((), device=DEV) * 0.7
    loss.backward(go if reduction == "none" else go.reshape(1))

    h, mask, ht = reference(inputs, "tanh", p, seed, (ranges, R) if pruned else None)
    _, _, ht_all = reference(inputs, "tanh", p, seed)
    if pruned:   # the eager pruned recipe: prune_joint_inputs -> act -> dropout with the cell's mask -> linear
        idx = (ranges.long()[..., None] + torch.arange(R, device=DEV)).clamp(0, U - 1)
        rows = ht_all[torch.arange(N, device=DEV)[:, None, None], torch.arange(T, device=DEV)[None, :, None], idx]
        logits = F.linear(rows.float(), weight.float(), bias.float()).detach().requires_grad_(True)
        ref = w.pruned_rnnt_loss(logits, labels, tl, ul, ranges, 0, reduction, delay_penalty=delay_penalty,
                                 rnnt_type=rnnt_type)
    else:
        logits = F.linear(ht.float(), weight.float(), bias.float()).detach().requires_grad_(True)
        ref = w.rnnt_loss(logits, labels, tl, ul, 0, reduction, delay_penalty=delay_penalty, rnnt_type=rnnt_type)
    ref.backward(go if reduction == "none" else go.reshape(1))

    if pruned:
        px_ref, py_ref = dr.pruned_log_probs(ht, weight, bias, labels, tl, ul, ranges, R)
    else:
        px_ref, py_ref = dr.log_probs(ht, weight, bias, labels, tl, ul)
    bar, _ = tg.factor_bar(ht, weight, bias, px_ref, py_ref)
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

    dl = logits.grad.double()
    if pruned:
        dl = tp.scatter_rows(dl, ranges, R, tl, ul, U)
        cov = pjr.covered(ranges, R, tl, ul, T, U)
    else:
        cov = jr.masks(tl, ul, T, U)[0]
    prob = torch.softmax(jr.logits(ht, weight, bias), -1) * cov[..., None]
    gsum = (gy.permute(0, 2, 1) + F.pad(gx.permute(0, 2, 1), (0, 1)))[..., None]
    onehots = jr.dlogits(ht, weight, bias, labels, tl, ul, gx, gy) + 2 * gsum * prob
    eps_occ = 3 * float(n.max()) * bmax + 4 * float(n.max()) * 2.0 ** -22
    err = 2.0 ** -8 * dl.abs() + eps_occ * (onehots + gsum * prob) + 4 * bar[..., None] * gsum * prob
    check_gradients([x.grad for x in leaves], ht, dr.act_grad(h, mask, p, "tanh"), weight, dl, err, 1)


@pytest.fixture
def no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


# 6. the seed's RNG behaviour

def _loss_and_grads(inputs, **kw):
    import warprnnt_pytorch as w
    enc, pred, weight, bias, labels, tl, ul = inputs
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    loss = w.joiner_rnnt_loss(*leaves, labels, tl, ul, 0, "sum", activation="relu", **kw)
    loss.backward()
    return [loss.detach()] + [x.grad for x in leaves]


def _same(a, b):
    return all(torch.equal(bits(x), bits(y)) for x, y in zip(a, b))


def test_seeds_reproduce_and_differ():
    inputs = tg.make(6, 3, 10, 5, 64, 100, nan_pad=False)
    a = _loss_and_grads(inputs, dropout=0.2, dropout_seed=seed_tensor(5))
    assert _same(a, _loss_and_grads(inputs, dropout=0.2, dropout_seed=seed_tensor(5)))
    assert not _same(a, _loss_and_grads(inputs, dropout=0.2, dropout_seed=seed_tensor(6)))
    torch.manual_seed(123)
    b = _loss_and_grads(inputs, dropout=0.2)
    c = _loss_and_grads(inputs, dropout=0.2)
    torch.manual_seed(123)
    assert _same(b, _loss_and_grads(inputs, dropout=0.2))
    assert not _same(b, c)


def test_checkpoint_recomputes_the_same_mask():
    import torch.utils.checkpoint as cp
    import warprnnt_pytorch as w
    enc, pred, weight, bias, labels, tl, ul = tg.make(7, 3, 10, 5, 64, 100, nan_pad=False)
    out = []
    for use_cp in (False, True):
        leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
        f = lambda e, q, wt, b: w.joiner_rnnt_loss(e, q, wt, b, labels, tl, ul, 0, "sum", activation="tanh",
                                                   dropout=0.2)
        torch.manual_seed(77)
        loss = cp.checkpoint(f, *leaves, use_reentrant=False) if use_cp else f(*leaves)
        loss.backward()
        out.append([loss.detach()] + [x.grad for x in leaves])
    assert _same(*out)


@pytest.mark.parametrize("pruned", [False, True])
def test_module_dropout_applies_in_training_only(pruned):
    import warprnnt_pytorch as w
    N, T, U = 3, 10, 5
    inputs = tg.make(8, N, T, U, 64, 100, nan_pad=False)
    enc, pred, weight, bias, labels, tl, ul = inputs
    extra = (tp.simple_ranges(2, inputs, 3), 3) if pruned else ()
    cls = w.PrunedJoinerRNNTLoss if pruned else w.JoinerRNNTLoss
    plain = cls(activation="relu")(enc, pred, weight, bias, labels, tl, ul, *extra)
    mod = cls(activation="relu", dropout=0.2)
    assert mod.training
    torch.manual_seed(1)
    train = mod(enc, pred, weight, bias, labels, tl, ul, *extra)
    torch.manual_seed(1)
    assert torch.equal(train, mod(enc, pred, weight, bias, labels, tl, ul, *extra))
    assert not torch.equal(train, plain)
    assert torch.equal(mod.eval()(enc, pred, weight, bias, labels, tl, ul, *extra), plain)


# 7. side streams and CUDA graphs

def test_side_stream_and_graph_capture():
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 3, 16, 6, 128, 200
    inputs = tg.make(8, N, T, U, H, V)
    enc, pred, weight, bias, labels, tl, ul = inputs
    seed = seed_tensor(0)

    def eager(s):
        r = run(inputs, 0, "tanh", 0.2, s, 100)
        return [r[0], r[1]] + r[4], r[2], r[3]

    expect, dpx, dpy = eager(31)

    def raw(px, py, ge, gp, gw, gb, ws, s):
        jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "tanh", 100, ws, dropout=0.2,
                              seed=s)
        jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, dpx, dpy, ge, gp, gw, gb, 0, "tanh", 100, ws,
                               dropout=0.2, seed=s)

    outs = [torch.empty_like(x) for x in expect]
    ws = torch.empty(jn.workspace_size(T, U, N, H, V, 100), dtype=torch.uint8, device=DEV)
    seed.fill_(31)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        raw(*outs, ws, seed)
    torch.cuda.current_stream().wait_stream(side)
    assert _same(outs, expect)

    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        raw(*outs, ws, seed)
    for s in (31, 32):   # the graph reads whatever seed the static tensor holds at replay
        seed.fill_(s)
        for o in outs:
            o.zero_()
        graph.replay()
        torch.cuda.synchronize()
        want, _, _ = eager(s) if s != 31 else (expect, None, None)
        assert _same(outs, want), s


def test_graph_replays_draw_fresh_seeds():
    """seed None draws the seed on the device from torch's CUDA generator (what the autograd Function does), so a
    captured draw gives every replay its own mask."""
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V = 3, 10, 5, 64, 100
    enc, pred, weight, bias, labels, tl, ul = tg.make(9, N, T, U, H, V)
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = torch.empty(jn.workspace_size(T, U, N, H, V), dtype=torch.uint8, device=DEV)
    jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "relu", None, ws, dropout=0.2,
                          seed=jn._seed_on(None, enc.device))   # warm-up outside capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        seed = jn._seed_on(None, enc.device)
        jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "relu", None, ws, dropout=0.2,
                              seed=seed)
    graph.replay()
    first = (py.clone(), seed.clone())
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(first[1], seed)
    assert not torch.equal(first[0][torch.isfinite(py)], py[torch.isfinite(py)])


# 8. launch counts

@pytest.mark.parametrize("pruned", [False, True])
@pytest.mark.parametrize("chunk_cells", [None, 64, 50])
def test_launch_counts(chunk_cells, pruned):
    import warprnnt_pytorch.joiner as jn
    N, T, U, H, V, R = 2, 10, 6, 64, 30, 3
    inputs = tg.make(4, N, T, U, H, V)
    enc, pred, weight, bias, labels, tl, ul = inputs
    window = dict(ranges=tp.simple_ranges(4, inputs, R), s_range=R) if pruned else {}
    chunks = tg.n_chunks(N, T, R if pruned else U, chunk_cells)
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, 0, "tanh", chunk_cells,
                               dropout=0.2, seed=seed_tensor(3), **window)
    assert jn.last_launch_count() == 2 * chunks + (1 if pruned else 0)
    g = [torch.empty_like(x) for x in (enc, pred, weight, bias)]
    jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, torch.zeros_like(px), torch.zeros_like(py), *g,
                           0, "tanh", chunk_cells, ws, dropout=0.2, seed=seed_tensor(3), **window)
    assert jn.last_launch_count() == 5 * chunks + 1
    torch.cuda.synchronize()
