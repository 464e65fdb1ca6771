"""The block-wise fp64 reference of the fused joiners (tests/joiner_blocks.py) and its plan() mirror, without a GPU:
the blocks give joiner_reference.py's factors and test_gpu_joiner.py's bars to fp64 roundoff (dense, pruned and with
dropout, over block sizes that do and do not divide the cell count), the mirror sizes the workspace as the library
does, and every shape of tests/test_gpu_joiner_scale.py runs the chunks, BM and slabs its comment claims."""
import numpy as np
import pytest
import torch

import dropout_reference as dr
import joiner_blocks as jb
import joiner_reference as jr
import pruned_joiner_reference as pjr
import test_gpu_joiner as tg
import test_gpu_joiner_scale as gs

I32_MAX = 2 ** 31 - 1


def make(seed, N, T, U, H, V, blank):
    """tg.make's inputs on the CPU: ragged lengths, T_b = 1 and S_b = 0 for utterance 2, NaN in padded rows."""
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(N, T, H, generator=g).to(torch.bfloat16)
    pred = torch.randn(N, U, H, generator=g).to(torch.bfloat16)
    weight = (torch.randn(V, H, generator=g) * (2.0 / H ** 0.5)).to(torch.bfloat16)
    bias = torch.randn(V, generator=g).to(torch.bfloat16)
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    labels[0, 1] = V + 3                      # outside the alphabet: NaN px
    tl = torch.randint(max(1, T // 2), T + 1, (N,), generator=g, dtype=torch.int32)
    ul = torch.randint(0, U, (N,), generator=g, dtype=torch.int32)
    tl[0], ul[0] = T, U - 1
    tl[2], ul[2] = 1, 0
    for i in range(N):
        enc[i, tl[i]:] = float('nan')
        pred[i, ul[i] + 1:] = float('nan')
    return [enc, pred, weight, bias, labels, tl, ul]


def ranges_of(seed, N, T, U, R):
    """Window starts: ordinary, negative, beyond S_b and +-(2^31 - 1)."""
    rng = np.random.default_rng(seed)
    r = rng.integers(-R, U + 1, (N, T))
    pick = rng.random((N, T))
    r = np.where(pick < 0.08, I32_MAX, np.where(pick > 0.92, -I32_MAX - 1, r))
    return torch.tensor(r, dtype=torch.int32)


def incoming(seed, inputs):
    """Random dpx, dpy with NaN on padding (tg.incoming on the CPU)."""
    enc, pred, _, _, _, tl, ul = inputs
    N, T, U = enc.shape[0], enc.shape[1], pred.shape[1]
    g = torch.Generator().manual_seed(seed)
    dpx, dpy = torch.randn(N, U - 1, T, generator=g), torch.randn(N, U, T, generator=g)
    cell, lab = jr.masks(tl, ul, T, U)
    dpy[~cell.permute(0, 2, 1)] = float('nan')
    dpx[~lab.permute(0, 2, 1)] = float('nan')
    return dpx, dpy


def full_reference(inputs, blank, activation, dpx, dpy, chunks, slabs, window, dropout):
    """joiner_reference / pruned_joiner_reference / dropout_reference on whole tensors, with test_gpu_joiner's
    factor_bar, dl_error and gradient_bars: what the GPU tests judge the kernels by at small sizes."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, H = enc.shape
    U = pred.shape[1]
    h = tg.reference_h(enc, pred, tl, ul, activation)
    if window is not None:
        h = h.masked_fill(~pjr.covered(*window, tl, ul, T, U)[..., None], 0)
    ht, ag = h, jr.act_grad(h, activation)
    if dropout is not None:
        mask = dr.keep_mask(dropout[1], N, T, U, H, dropout[0])
        ht, ag = dr.dropped_hidden(h, mask, dropout[0]), dr.act_grad(h, mask, dropout[0], activation)
    if window is None:
        px, py = jr.log_probs(ht, weight, bias, labels, tl, ul, blank)
        cov = jr.masks(tl, ul, T, U)[0]
        gx, gy = torch.nan_to_num(dpx, nan=0.0), torch.nan_to_num(dpy, nan=0.0)   # padding is not read
    else:
        px, py = pjr.log_probs(ht, weight, bias, labels, tl, ul, *window, blank)
        cov = pjr.covered(*window, tl, ul, T, U)
        gx, gy = pjr.masked_incoming(dpx, dpy, *window, tl, ul)
    bar, lse = tg.factor_bar(ht, weight, bias, px, py)
    dl = jr.dlogits(ht, weight, bias, labels, tl, ul, gx, gy, blank)
    err = tg.dl_error(ht, weight, bias, dl, gx, gy, tl, ul, bar)
    ref, bars = tg.gradient_bars(ht, ag, weight, dl, err, chunks, slabs)
    return px, py, bar, lse, cov, ref, bars


def same(a, b, what):
    assert a.shape == b.shape, what
    inf, nan = torch.isinf(b), torch.isnan(b)
    assert torch.equal(torch.isinf(a), inf) and torch.equal(a[inf], b[inf]), what
    assert torch.equal(torch.isnan(a), nan), what
    ok = ~(inf | nan)
    torch.testing.assert_close(a[ok], b[ok], rtol=1e-12, atol=1e-14, msg=what)


@pytest.mark.parametrize("block", ["one", "divides", "ragged"])
@pytest.mark.parametrize("kind", ["dense", "pruned", "dropout", "pruned-dropout"])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_blocks_equal_the_full_tensor_reference(activation, kind, block):
    N, T, U, H, V, R = 4, 9, 6, 32, 70, 3
    blank = 0 if activation == "tanh" else V - 1
    inputs = make(len(kind) + H, N, T, U, H, V, blank)
    window = (ranges_of(len(kind), N, T, U, R), R) if "pruned" in kind else None
    dropout = (0.3, -987654321012) if "dropout" in kind else None
    dpx, dpy = incoming(5, inputs)
    chunks, slabs = 3, 2
    n = len(jb.cells(inputs, window)[0])
    step = {"one": n, "divides": next(d for d in range(7, n) if n % d == 0),
            "ragged": next(d for d in range(7, n) if n % d)}[block]
    got = jb.reference(inputs, blank, activation, dpx, dpy, chunks, slabs, window, dropout, block=step)
    px, py, bar, lse, cov, ref, bars = full_reference(inputs, blank, activation, dpx, dpy, chunks, slabs, window,
                                                      dropout)
    assert torch.isnan(px).any() and torch.isinf(px).any()
    same(got.px, px, "px")
    same(got.py, py, "py")
    same(got.lse[cov], lse[cov], "lse")
    same(got.bar[cov], bar[cov], "factor bar")
    for name, a, b in zip(("d_enc", "d_pred", "d_weight", "d_bias"), got.grads, ref):
        same(a, b, name)
    for name, a, b in zip(("d_enc", "d_pred", "d_weight", "d_bias"), got.bars, bars):
        same(a, b, name + " bar")


def test_grid_rows_decode_the_chunk_rows():
    """Dense rows (b, u, t) and pruned rows (b, r, t), t fastest, as the kernels' decode() enumerates them."""
    N, T, U, R = 3, 5, 4, 2
    inputs = make(1, N, T, U, 16, 10, 0)
    tl, ul = inputs[5], inputs[6]
    valid, b, t, u = jb.grid_rows(inputs, 0, N * T * U)
    cell = jr.masks(tl, ul, T, U)[0]
    assert torch.equal(valid.view(N, U, T), cell.permute(0, 2, 1))
    assert torch.equal(b.view(N, U, T)[:, 0, 0], torch.arange(N))
    assert torch.equal(t.view(N, U, T)[0, 0], torch.arange(T))
    assert torch.equal(u.view(N, U, T)[0, :, 0], torch.arange(U))        # utterance 0 is full
    ranges = ranges_of(3, N, T, U, R)
    valid, b, t, u = jb.grid_rows(inputs, 0, N * T * R, (ranges, R))
    cov = torch.zeros(N, T, U, dtype=torch.bool)
    cov[b[valid], t[valid], u[valid]] = True
    assert torch.equal(cov, pjr.covered(ranges, R, tl, ul, T, U))
    assert int(valid.sum()) == int(cov.sum())            # no cell is covered twice


def _gpu_calls():
    """(T, U, N, H, V, chunk_cells, s_range) of every call tests/test_gpu_joiner_scale.py makes."""
    out = []
    for c in gs.SCALE.values():
        N, T, U, H, V = c["shape"]
        out.append((T, U, N, H, V, None, c["R"]))
    N, T, U, H, V = gs.SCALE["D1"]["shape"]
    out += [(T, U, N, H, V, None, d["R"]) for d in gs.DROPOUT.values()]
    N, T, U = gs.WIDTH_SHAPE
    out += [(T, U, N, H, V, ch, None) for H in gs.WIDTHS for V in (64, 1000) for ch in (None, gs.SMALL_CHUNK)]
    N, T, U, H = gs.FULL_TILE_SHAPE
    out += [(T, U, N, H, V, ch, None) for V, _ in gs.FULL_TILE for ch in (None, gs.SMALL_CHUNK)]
    return out


# beyond the GPU file's shapes: a chunk cap below one wave, a cap below one 128-row CTA, explicit chunks, R > U
EXTRA = [(50, 11, 8, 1024, 100000, None, None), (4, 3, 2, 16, 2000000, None, None), (13, 7, 4, 64, 500, 37, None),
         (70, 9, 4, 64, 500, 1000, 4), (11, 5, 5, 128, 300, None, 9), (150, 21, 128, 640, 5000, None, 5)]


@pytest.mark.parametrize("call", _gpu_calls() + EXTRA)
def test_plan_mirror_sizes_the_workspace_as_the_library(call):
    import warprnnt_pytorch.joiner as jn
    T, U, N, H, V, chunk, R = call
    assert jn.workspace_size(T, U, N, H, V, chunk, R) == jb.plan(T, U, N, H, V, chunk, R).bytes


def test_scale_cases_run_the_plan_they_claim():
    for name, c in gs.SCALE.items():
        N, T, U, H, V = c["shape"]
        p = jb.plan(T, U, N, H, V, None, c["R"])
        assert {k: getattr(p, k) for k in c["plan"]} == c["plan"], name
        assert p.chunks > 1 and 0 < p.last < p.chunk, name            # several default chunks, a ragged last one
    for name in ("D3", "P1"):
        N, T, U, H, V = gs.SCALE[name]["shape"]
        p = jb.plan(T, U, N, H, V, None, gs.SCALE[name]["R"])
        assert p.Vp == V and V // 64 == 500, name                       # 500 k-tiles, no masked column
        assert p.slabs == 1 and p.chunk > 64 * 50, name                 # one slab over many row tiles
    assert gs.SCALE["D3"]["blank"] == gs.SCALE["D3"]["shape"][4] - 1
    N, T, U, H, V = gs.SCALE["D1"]["shape"]
    for d in gs.DROPOUT.values():
        p = jb.plan(T, U, N, H, V, None, d["R"])
        assert {k: getattr(p, k) for k in d["plan"]} == d["plan"]


def test_width_cases_have_a_partial_last_k_tile_on_both_sides_of_bm():
    N, T, U = gs.WIDTH_SHAPE
    bms = set()
    for H in gs.WIDTHS:
        assert H % 16 == 0 and H % 64 and H > 64, H                    # more than one k-tile, the last partial
        for V in (64, 1000):
            assert jb.plan(T, U, N, H, V).chunks == 1
            p = jb.plan(T, U, N, H, V, gs.SMALL_CHUNK)
            assert p.chunks > 1 and p.chunk % 64 and p.last % 64, (H, V)   # chunk edges inside a 64-row tile
            bms.add(p.bm)
    assert bms == {64, 128}
    assert jb.plan(T, U, N, 656, 64).bm == 64 and jb.plan(T, U, N, 640, 64).bm == 128


def test_full_tile_cases_have_no_masked_column():
    for V, blank in gs.FULL_TILE:
        N, T, U, H = gs.FULL_TILE_SHAPE
        assert jb.plan(T, U, N, H, V).Vp == V and blank % 64 == 63
