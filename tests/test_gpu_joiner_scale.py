"""The fused and pruned fused joiners (DESIGN.md §14-§16) at the sizes production calls run, against the block-wise
fp64 reference (tests/joiner_blocks.py) with test_gpu_joiner.py's per-element bars and no floor:

- several default-size chunks with a ragged last one, where the logits grid spans many CTA waves;
- one dW slab folding tens of thousands of rows per chunk, chunk after chunk;
- V 32 000: 500 k-tiles in the ds contraction and 500 column tiles of online max / sum, with Vp == V;
- widths with a partial last k-tile on both sides of the logits kernels' 128 / 64-row switch (H 640);
- a full last W tile with the blank and labels in its edge columns;
- dropout at the default chunk, dense and pruned.

Beyond the outputs, each call checks the stages the workspace still holds afterwards against fp64 on their own
operands: the lse of every row (it persists across chunks), and the last chunk's h (bit for bit torch's h, or h~),
bf16 dlogits (under dl_error) and fp32 ds (against the kernel's own dlogits times W and act', under the ds contraction
term alone).  The plan each case claims (chunk count, last chunk, BM, slabs) is checked on the CPU by
tests/test_joiner_blocks.py.  Each call prints its worst error / bar ratio per quantity."""
import json

import pytest
import torch

import joiner_blocks as jb
import test_gpu_joiner as tg
import test_gpu_pruned_joiner as tp

pytestmark = pytest.mark.gpu

DEV = "cuda"
U_ = 2.0 ** -24

# (N, T, U, H, V), activation, blank, R (None: dense), and what plan() runs at the default chunk
SCALE = {
    "D1": dict(shape=(16, 250, 30, 512, 500), act="tanh", blank=0, R=None,
               plan=dict(chunks=3, chunk=50688, last=18624, bm=128, slabs=4)),
    "D2": dict(shape=(4, 150, 61, 1024, 5000), act="relu", blank=0, R=None,
               plan=dict(chunks=3, chunk=16384, last=3832, bm=64, slabs=1)),
    "D3": dict(shape=(2, 100, 45, 640, 32000), act="tanh", blank=31999, R=None,
               plan=dict(chunks=3, chunk=3840, last=1320, bm=128, slabs=1)),
    "P1": dict(shape=(4, 500, 101, 640, 32000), act="relu", blank=0, R=5,
               plan=dict(chunks=3, chunk=3840, last=2320, bm=128, slabs=1)),
}
# D1's shape with dropout 0.2: dense (3 chunks) and pruned with R 5 (20 000 rows: one chunk, 4 slabs)
DROPOUT = {"dense": dict(R=None, plan=dict(chunks=3, chunk=50688, last=18624, bm=128, slabs=4)),
           "pruned": dict(R=5, plan=dict(chunks=1, chunk=20000, last=20000, bm=128, slabs=4))}
# widths with a partial last k-tile (H % 64 != 0, more than one k-tile), BM 128 for H <= 640 and 64 above, at a small
# cell count, with the default chunk and with a chunk that ends inside a 64-row tile
WIDTHS = [80, 528, 656, 1008]
WIDTH_SHAPE = (4, 23, 7)
SMALL_CHUNK = 100
# V a multiple of 64: the last W tile is full, no column is masked
FULL_TILE = [(64, 63), (512, 511), (512, 63)]
FULL_TILE_SHAPE = (4, 17, 9, 128)


def make(seed, N, T, U, H, V, blank=0, scale=1.0):
    """test_gpu_joiner.make's inputs with the last utterance full, so the last chunk (the one whose stages the
    workspace keeps) holds valid rows."""
    inputs = tg.make(seed, N, T, U, H, V, blank, scale=scale)
    g = torch.Generator().manual_seed(seed + 1)
    inputs[0][-1] = (torch.randn(T, H, generator=g) * scale).to(torch.bfloat16).to(DEV)
    inputs[1][-1] = (torch.randn(U, H, generator=g) * scale).to(torch.bfloat16).to(DEV)
    inputs[5][-1], inputs[6][-1] = T, U - 1
    return inputs


def seed_tensor(s):
    return torch.tensor([s], dtype=torch.int64, device=DEV)


def bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


def call(inputs, blank, activation, chunk_cells=None, window=None, dropout=None, grad_seed=0):
    """Forward and backward through the C-ABI, as the autograd Function runs them, keeping the workspace."""
    import warprnnt_pytorch.joiner as jn
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, _ = enc.shape
    U = pred.shape[1]
    kw = dict(ranges=window[0], s_range=window[1]) if window else {}
    if dropout:
        kw.update(dropout=dropout[0], seed=seed_tensor(dropout[1]))
    px = torch.empty(N, U - 1, T, device=DEV)
    py = torch.empty(N, U, T, device=DEV)
    ws = jn.gpu_joiner_forward(enc, pred, weight, bias, labels, tl, ul, px, py, blank, activation, chunk_cells, **kw)
    if window:
        dpx, dpy = tp.incoming(grad_seed, px, py, *window, tl, ul)
    else:
        dpx, dpy = tg.incoming(grad_seed, px, py, tl, ul)
    grads = [torch.empty_like(x) for x in (enc, pred, weight, bias)]
    jn.gpu_joiner_backward(enc, pred, weight, bias, labels, tl, ul, dpx, dpy, *grads, blank, activation, chunk_cells,
                           ws, **kw)
    torch.cuda.synchronize()
    return px, py, dpx, dpy, grads, ws


def factor_ratios(px, py, ref):
    """test_gpu_joiner.check_factors, returning the worst error / bar of px and py."""
    out = []
    for name, got, r, b in (("px", px, ref.px, ref.bar[:, :, :-1].permute(0, 2, 1)),
                            ("py", py, ref.py, ref.bar.permute(0, 2, 1))):
        inf, nan = torch.isinf(r), torch.isnan(r)
        assert torch.equal(got[inf], r[inf].float()), name + ": padding must be -inf"
        assert torch.isnan(got[nan]).all(), name
        ok = ~(inf | nan)
        out.append(jb.ratio(name, got[ok], r[ok], b[ok]))
    return out


def stages(ws, p, inputs, blank, activation, dpx, dpy, window, dropout, ref):
    """The lse of every row, and the last chunk's h, dlogits and ds, read from the workspace after the backward."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    H, V = p.H, p.V
    out = {}
    valid, b, t, u = jb.grid_rows(inputs, 0, p.cells, window)
    lse = ws[p.lse:p.lse + p.cells * 4].view(torch.float32)
    assert (lse[~valid] == 0).all(), "padding rows' lse"
    b, t, u = b[valid], t[valid], u[valid]
    out["lse"] = jb.ratio("lse", lse[valid], ref.lse[b, t, u], ref.bar[b, t, u])

    c0, m = (p.chunks - 1) * p.chunk, p.last
    valid, b, t, u = jb.grid_rows(inputs, c0, c0 + m, window)
    h = ws[p.h:p.h + m * p.Hp * 2].view(torch.bfloat16).view(m, p.Hp)
    dlog = ws[p.dlog:p.dlog + m * p.Vp * 2].view(torch.bfloat16).view(m, p.Vp)
    ds = ws[p.ds:p.ds + m * H * 4].view(torch.float32).view(m, H)
    assert (h[:, H] == 1).all() and (h[:, H + 1:] == 0).all(), "h columns H (1) and past it (0)"
    assert (h[~valid, :H] == 0).all() and (dlog[~valid] == 0).all(), "padding rows of h and dlogits"
    assert (dlog[:, V:] == 0).all(), "dlogits past V"
    rows = valid.nonzero(as_tuple=True)[0]
    assert len(rows), "the last chunk has no valid row to check"
    b, t, u = b[rows], t[rows], u[rows]
    wd, wa = weight.double(), weight.double().abs()
    g_ds = (32 + V / 256) * 2 * U_
    out["dlogits"] = out["ds"] = 0.0
    flips = 0
    step = jb.block_rows(V)
    for i in range(0, len(rows), step):
        r = rows[i:i + step]
        x = jb.terms(inputs, b[i:i + step], t[i:i + step], u[i:i + step], blank, activation, dpx, dpy, dropout)
        flips += int((bits(h[r, :H]) != bits(x.ht)).sum())
        dk = dlog[r, :V].double()
        out["dlogits"] = max(out["dlogits"], jb.ratio("dlogits", dk, x.dl, x.dl_err))
        out["ds"] = max(out["ds"], jb.ratio("ds", ds[r], (dk @ wd) * x.ag, g_ds * (dk.abs() @ wa) * x.ag))
        del x, dk
    assert flips == 0, "%d h elements of the last chunk differ from torch's" % flips
    return out


def check(case, inputs, blank, activation, chunk_cells=None, window=None, dropout=None, expect=None):
    """One call against the block-wise reference; returns and prints the worst error / bar per quantity."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, H = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    p = jb.plan(T, U, N, H, V, chunk_cells, window[1] if window else None)
    if expect:
        assert {k: getattr(p, k) for k in expect} == expect
    sel = None
    if window:
        inputs, sel = tp.nan_unselected_pred(inputs, *window)
    torch.cuda.reset_peak_memory_stats()
    px, py, dpx, dpy, grads, ws = call(inputs, blank, activation, chunk_cells, window, dropout)
    assert ws.numel() == p.bytes
    ref = jb.reference(inputs, blank, activation, dpx, dpy, p.chunks, p.slabs, window, dropout)
    out = dict(chunks=p.chunks, bm=p.bm, slabs=p.slabs)
    out["px"], out["py"] = factor_ratios(px, py, ref)
    out.update(zip(("d_enc", "d_pred", "d_weight", "d_bias"), jb.gradient_ratios(grads, ref.grads, ref.bars)))
    for i in range(N):
        assert (grads[0][i, tl[i]:] == 0).all() and (grads[1][i, ul[i] + 1:] == 0).all(), "padding rows"
    if sel is not None:
        assert (grads[1][~sel] == 0).all(), "pred rows no valid row selects"
    out.update(stages(ws, p, inputs, blank, activation, dpx, dpy, window, dropout, ref))
    out["peak_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    print("joiner-scale", case, json.dumps({k: round(v, 4) if isinstance(v, float) else v for k, v in out.items()}))
    return out


def scale_inputs(name):
    c = SCALE[name]
    N, T, U, H, V = c["shape"]
    inputs = make(sum(c["shape"]), N, T, U, H, V, c["blank"])
    window = (tp.simple_ranges(V, inputs, c["R"]), c["R"]) if c["R"] else None
    return c, inputs, window


@pytest.mark.parametrize("name", list(SCALE))
def test_default_chunks_at_scale(name):
    c, inputs, window = scale_inputs(name)
    check(name, inputs, c["blank"], c["act"], window=window, expect=c["plan"])


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("kind", list(DROPOUT))
def test_dropout_at_the_default_chunk(kind, activation):
    c = SCALE["D1"]
    N, T, U, H, V = c["shape"]
    inputs = make(71, N, T, U, H, V)
    R = DROPOUT[kind]["R"]
    window = (tp.simple_ranges(72, inputs, R), R) if R else None
    check("DR-%s-%s" % (kind, activation), inputs, 0, activation, window=window, dropout=(0.2, 2 ** 35 + 17),
          expect=DROPOUT[kind]["plan"])


@pytest.mark.parametrize("chunk_cells", [None, SMALL_CHUNK])
@pytest.mark.parametrize("V", [64, 1000])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("H", WIDTHS)
def test_widths_with_a_partial_last_k_tile(H, activation, V, chunk_cells):
    N, T, U = WIDTH_SHAPE
    blank = 0 if V == 64 else V - 1
    inputs = make(H + V, N, T, U, H, V, blank, scale=1.5)
    check("H%d-%s-V%d-%s" % (H, activation, V, chunk_cells), inputs, blank, activation, chunk_cells)


def full_tile_labels(inputs, V):
    """Labels cycling through 0, 63, 64 and V - 1 (those inside the alphabet)."""
    labels = inputs[4]
    edge = torch.tensor([x for x in (0, 63, 64, V - 1) if x < V], dtype=torch.int32, device=DEV)
    N, S = labels.shape
    idx = (torch.arange(N, device=DEV)[:, None] + torch.arange(S, device=DEV)[None, :]) % len(edge)
    inputs[4] = edge[idx].contiguous()
    return inputs


@pytest.mark.parametrize("chunk_cells", [None, SMALL_CHUNK])
@pytest.mark.parametrize("V, blank", FULL_TILE)
def test_full_last_tile(V, blank, chunk_cells):
    N, T, U, H = FULL_TILE_SHAPE
    inputs = full_tile_labels(make(V + blank, N, T, U, H, V, blank), V)
    activation = "tanh" if blank == V - 1 else "relu"
    check("V%d-blank%d-%s" % (V, blank, chunk_cells), inputs, blank, activation, chunk_cells)


def test_deterministic_at_the_default_chunk():
    c, inputs, _ = scale_inputs("D1")
    a = call(inputs, c["blank"], c["act"])
    b = call(inputs, c["blank"], c["act"])
    for x, y in zip([a[0], a[1]] + a[4], [b[0], b[1]] + b[4]):
        assert torch.equal(bits(x), bits(y))
