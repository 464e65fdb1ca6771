"""The fp64 joiner reference (tests/joiner_reference.py) against the dense references on its materialised logits, fp64
autograd and gradcheck.  CPU only."""
import numpy as np
import pytest
import torch

import delay_reference as dr
import joiner_reference as jr
import lattice_reference as lr


def _inputs(seed, N=3, T=5, U=4, H=16, V=7, bias=True, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(N, T, H, generator=g).to(dtype)
    pred = torch.randn(N, U, H, generator=g).to(dtype)
    weight = (torch.randn(V, H, generator=g) / H ** 0.5).to(dtype)
    b = torch.randn(V, generator=g).to(dtype) if bias else None
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    act_lens = torch.tensor([T] + [max(1, T - 1 - i) for i in range(N - 1)], dtype=torch.int32)
    label_lens = torch.tensor([U - 1] + [(i % U) for i in range(N - 1)], dtype=torch.int32)
    return enc, pred, weight, b, labels, act_lens, label_lens


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("blank", [0, 6])
@pytest.mark.parametrize("delay_penalty", [0.0, 0.3])
def test_costs_match_the_dense_reference_on_materialised_logits(activation, blank, delay_penalty):
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(1 + blank)
    h = jr.hidden(enc, pred, activation)
    z = jr.logits(h, weight, bias).numpy()
    px, py = jr.log_probs(h, weight, bias, labels, act_lens, label_lens, blank)
    gx, gy = lr.factors_from_logits(z, labels.numpy(), blank)
    cell, lab = jr.masks(act_lens, label_lens, h.shape[1], h.shape[2])
    np.testing.assert_allclose(py.numpy()[cell.permute(0, 2, 1).numpy()], gy[cell.permute(0, 2, 1).numpy()],
                               rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(px.numpy()[lab.permute(0, 2, 1).numpy()], gx[lab.permute(0, 2, 1).numpy()],
                               rtol=1e-13, atol=1e-13)
    assert np.all(py.numpy()[~cell.permute(0, 2, 1).numpy()] == -np.inf)
    assert np.all(px.numpy()[~lab.permute(0, 2, 1).numpy()] == -np.inf)
    T = h.shape[1]
    tb = act_lens.numpy().clip(1, T)
    pen = delay_penalty * ((tb[:, None, None] - 1) / 2.0 - np.arange(T)[None, None, :])
    costs, _, _ = lr.loss(px.numpy() + pen, py.numpy(), act_lens.numpy(), label_lens.numpy())
    ref, _ = dr.loss(z, labels.numpy(), act_lens.numpy(), label_lens.numpy(), blank=blank,
                     delay_penalty=delay_penalty)
    np.testing.assert_allclose(costs, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("activation", ["tanh", "relu"])
@pytest.mark.parametrize("bias", [True, False])
def test_explicit_gradients_are_fp64_autograd(activation, bias):
    enc, pred, weight, b, labels, act_lens, label_lens = _inputs(7, bias=bias, dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in (enc, pred, weight)] + \
             ([b.clone().requires_grad_(True)] if bias else [None])
    px, py = jr.fp64_forward(*leaves, labels, act_lens, label_lens, activation, blank=2)
    g = torch.Generator().manual_seed(3)
    dpx, dpy = torch.randn(px.shape, generator=g, dtype=torch.float64), torch.randn(py.shape, generator=g,
                                                                                    dtype=torch.float64)
    fin_x, fin_y = torch.isfinite(px), torch.isfinite(py)
    zx, zy = px.where(fin_x, torch.zeros_like(px)), py.where(fin_y, torch.zeros_like(py))
    ((zx * dpx).sum() + (zy * dpy).sum()).backward()
    s = enc[:, :, None, :] + pred[:, None, :, :]
    h = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    de, dp, dw, db = jr.gradients(h, weight, b, labels, act_lens, label_lens, dpx, dpy, activation, blank=2)
    for got, ref in ((de, leaves[0].grad), (dp, leaves[1].grad), (dw, leaves[2].grad)):
        torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    if bias:
        torch.testing.assert_close(db, leaves[3].grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_fp64_form_passes_gradcheck(activation):
    enc, pred, weight, b, labels, act_lens, label_lens = _inputs(11, N=2, T=3, U=3, H=16, V=5, dtype=torch.float64)
    if activation == 'relu':   # keep every pre-activation away from the kink
        enc = enc + torch.sign(enc) * 0.1

    def f(e, p, w, bb):
        px, py = jr.fp64_forward(e, p, w, bb, labels, act_lens, label_lens, activation)
        fin_x, fin_y = torch.isfinite(px), torch.isfinite(py)
        return px[fin_x], py[fin_y]

    args = [t.clone().requires_grad_(True) for t in (enc, pred, weight, b)]
    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-7)


def test_label_outside_the_alphabet_gives_nan_on_its_row_only():
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(5)
    labels[0, 1] = weight.shape[0] + 3
    h = jr.hidden(enc, pred, 'tanh')
    px, py = jr.log_probs(h, weight, bias, labels, act_lens, label_lens)
    assert torch.isnan(px[0, 1]).all()
    px[0, 1] = 0
    assert not torch.isnan(px).any() and not torch.isnan(py).any()
