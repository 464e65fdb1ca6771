"""The dropout reference (tests/dropout_reference.py): Philox4x32-10 against Random123's known answers, the keep
mask's statistics, and the fp64 gradients with a fixed mask against fp64 autograd and gradcheck, dense and pruned.
CPU only."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_reference as dr
import joiner_reference as jr
import pruned_joiner_reference as pjr


def _hex(words):
    return ["%08x" % int(w) for w in words]


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    assert _hex(dr.philox4x32_10((0, 0, 0, 0), (0, 0))) == ["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"]
    ones = 0xFFFFFFFF
    assert _hex(dr.philox4x32_10((ones,) * 4, (ones,) * 2)) == ["408f276d", "41c83b0e", "a20bc7c6", "6d5451fd"]
    assert _hex(dr.philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0))) == \
        ["d16cfe09", "94fdcceb", "5001e420", "24126ea1"]


def test_philox_is_elementwise():
    ctr = (np.arange(5), np.array([7]), 0, 0)
    words = dr.philox4x32_10(ctr, (3, 9))
    for i in range(5):
        assert [int(w[i]) for w in words] == [int(w) for w in dr.philox4x32_10((i, 7, 0, 0), (3, 9))]


def test_mask_layout():
    """Element k of cell (b, t, u) is word k & 3 of counter (k >> 2, (b U + u) T + t)."""
    N, T, U, H, p, seed = 2, 3, 4, 16, 0.3, -12345
    m = dr.keep_mask(seed, N, T, U, H, p)
    thr = dr.threshold(p)
    key = dr.seed_key(seed)
    for b, t, u, k in [(0, 0, 0, 0), (1, 2, 3, 15), (1, 0, 2, 6), (0, 2, 1, 9)]:
        x = dr.philox4x32_10((k >> 2, (b * U + u) * T + t, 0, 0), key)[k & 3]
        assert bool(m[b, t, u, k]) == (int(x) >= thr)
    assert key == ((-12345) & 0xFFFFFFFF, ((-12345) & (2 ** 64 - 1)) >> 32)


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_keep_fraction_is_binomial(p):
    N, T, U, H = 2, 20, 6, 64
    n = N * T * U * H
    q = 1 - dr.threshold(p) / 2.0 ** 32
    for seed in (0, 1, 2 ** 40 + 7, -1):
        kept = int(dr.keep_mask(seed, N, T, U, H, p).sum())
        assert abs(kept - n * q) <= 5 * math.sqrt(n * q * (1 - q)), (seed, kept, n * q)


def test_distinct_seeds_give_distinct_masks_and_p0_keeps_everything():
    masks = [dr.keep_mask(s, 2, 5, 3, 32, 0.2) for s in (0, 1, 2, 2 ** 32, -1)]
    for i in range(len(masks)):
        for j in range(i):
            assert not torch.equal(masks[i], masks[j]), (i, j)
    assert dr.keep_mask(5, 2, 5, 3, 32, 0.0).all()
    assert dr.threshold(0.0) == 0 and dr.scale(0.0) == 1.0


def test_threshold_and_scale_follow_the_float32_p():
    assert dr.threshold(0.5) == 2 ** 31
    p32 = float(np.float32(0.2))
    assert dr.threshold(0.2) == math.floor(p32 * 2 ** 32)
    assert dr.scale(0.2) == float(np.float32(1 / (1 - p32)))


def test_dropped_hidden():
    g = torch.Generator().manual_seed(0)
    h = torch.randn(2, 3, 4, 16, generator=g).to(torch.bfloat16)
    m = dr.keep_mask(9, 2, 3, 4, 16, 0.2)
    ht = dr.dropped_hidden(h, m, 0.2)
    assert (ht[~m] == 0).all()
    assert torch.equal(ht[m], (h.float()[m] * dr.scale(0.2)).to(torch.bfloat16))


def _inputs(seed, N=3, T=4, U=3, H=16, V=6):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(N, T, H, generator=g, dtype=torch.float64)
    pred = torch.randn(N, U, H, generator=g, dtype=torch.float64)
    weight = torch.randn(V, H, generator=g, dtype=torch.float64) / H ** 0.5
    bias = torch.randn(V, generator=g, dtype=torch.float64)
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    act_lens = torch.tensor([T] + [max(1, T - 1 - i) for i in range(N - 1)], dtype=torch.int32)
    label_lens = torch.tensor([U - 1] + [i % U for i in range(N - 1)], dtype=torch.int32)
    return enc, pred, weight, bias, labels, act_lens, label_lens


def _fixed_dropout_forward(enc, pred, weight, bias, labels, act_lens, label_lens, activation, mask, p, blank):
    """linear(dropout_fixed(act(s))) in fp64, through log_softmax to (px, py), differentiable by autograd."""
    s = enc[:, :, None, :] + pred[:, None, :, :]
    h = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    z = F.linear(h * mask.double() * dr.scale(p), weight, bias)
    N, T, U, V = z.shape
    lp = torch.log_softmax(z, -1)
    cell, lab = jr.masks(act_lens, label_lens, T, U)
    py = torch.where(cell, lp[..., blank], torch.full_like(lp[..., blank], -float('inf')))
    g = lp[:, :, :U - 1, :].gather(-1, labels.long()[:, None, :, None].expand(N, T, U - 1, 1))[..., 0]
    px = torch.where(lab, g, torch.full_like(g, -float('inf')))
    return px.permute(0, 2, 1), py.permute(0, 2, 1), h


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("pruned", [False, True])
def test_gradients_are_fp64_autograd(activation, pruned):
    """The explicit gradients (h~ as the logits' operand, act' keep scale for ds) of a fixed mask, with h in fp64
    (no rounding), against autograd through linear(dropout_fixed(act(s))); pruned: the dense gradients of the
    incoming gradients masked to the covered cells."""
    p, blank = 0.3, 2
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(5)
    N, T, H = enc.shape
    U = pred.shape[1]
    mask = dr.keep_mask(77, N, T, U, H, p)
    leaves = [x.clone().requires_grad_(True) for x in (enc, pred, weight, bias)]
    px, py, h = _fixed_dropout_forward(*leaves, labels, act_lens, label_lens, activation, mask, p, blank)
    ranges = torch.tensor([[0, 1, 1, 2], [0, 0, 1, -1], [1, 0, 0, 0]], dtype=torch.int32)
    mx, my = pjr.factor_masks(ranges, 2, act_lens, label_lens, T, U) if pruned else \
        (torch.isfinite(px.detach()), torch.isfinite(py.detach()))
    g = torch.Generator().manual_seed(1)
    dpx = torch.randn(px.shape, generator=g, dtype=torch.float64)
    dpy = torch.randn(py.shape, generator=g, dtype=torch.float64)
    ((px.where(mx, torch.zeros_like(px)) * dpx).sum() + (py.where(my, torch.zeros_like(py)) * dpy).sum()).backward()
    h = h.detach()
    ht = h * mask.double() * dr.scale(p)
    if pruned:
        dpx[~mx], dpy[~my] = float('nan'), float('nan')   # off the covered cells: never read
        got = dr.pruned_gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, dpx, dpy, ranges, 2,
                                  activation, blank)
    else:
        got = dr.gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, torch.nan_to_num(dpx),
                           torch.nan_to_num(dpy), activation, blank)
    for x, leaf in zip(got, leaves):
        torch.testing.assert_close(x, leaf.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_fixed_mask_form_passes_gradcheck(activation):
    p = 0.5
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(11, N=2, T=3, U=3, H=16, V=5)
    if activation == 'relu':   # keep every pre-activation away from the kink
        enc = enc + torch.sign(enc) * 0.1
    mask = dr.keep_mask(3, 2, 3, 3, 16, p)
    assert not mask.all() and mask.any()

    def f(e, q, w, b):
        px, py, _ = _fixed_dropout_forward(e, q, w, b, labels, act_lens, label_lens, activation, mask, p, 0)
        return px[torch.isfinite(px)], py[torch.isfinite(py)]

    args = [t.clone().requires_grad_(True) for t in (enc, pred, weight, bias)]
    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-7)


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_pruned_reference_is_the_dense_one_masked(activation):
    g = torch.Generator().manual_seed(4)
    N, T, U, H, V, p = 3, 5, 4, 16, 7, 0.2
    enc = torch.randn(N, T, H, generator=g).to(torch.bfloat16)
    pred = torch.randn(N, U, H, generator=g).to(torch.bfloat16)
    weight = (torch.randn(V, H, generator=g) / 4).to(torch.bfloat16)
    bias = torch.randn(V, generator=g).to(torch.bfloat16)
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    act_lens = torch.tensor([T, 3, 1], dtype=torch.int32)
    label_lens = torch.tensor([U - 1, 2, 0], dtype=torch.int32)
    ranges = torch.tensor([[0, 0, 1, 1, 2], [0, 1, 1, 2, 2], [0, 0, 0, 0, 0]], dtype=torch.int32)
    h = jr.hidden(enc, pred, activation)
    mask = dr.keep_mask(2 ** 33 + 5, N, T, U, H, p)
    ht = dr.dropped_hidden(h, mask, p)
    dense = dr.log_probs(ht, weight, bias, labels, act_lens, label_lens)
    pruned = dr.pruned_log_probs(ht, weight, bias, labels, act_lens, label_lens, ranges, 2)
    for m, d, q in zip(pjr.factor_masks(ranges, 2, act_lens, label_lens, T, U), dense, pruned):
        assert torch.equal(q[m], d[m]) and torch.isneginf(q[~m]).all()
    full = dr.pruned_log_probs(ht, weight, bias, labels, act_lens, label_lens, torch.zeros_like(ranges), U)
    for a, b in zip(full, dense):
        assert torch.equal(a, b)
    gx = torch.randn(N, U - 1, T, generator=g, dtype=torch.float64)
    gy = torch.randn(N, U, T, generator=g, dtype=torch.float64)
    mx, my = pjr.factor_masks(ranges, 2, act_lens, label_lens, T, U)
    got = dr.pruned_gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, gx, gy, ranges, 2,
                              activation)
    ref = dr.gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, gx.where(mx, 0.0),
                       gy.where(my, 0.0), activation)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
