"""The fp64 pruned-joiner reference (tests/pruned_joiner_reference.py) against prune_joint_inputs -> the fp64 joiner
-> the pruned loss reference (tests/pruned_reference.py), fp64 autograd and gradcheck, on ordinary and adversarial
windows.  CPU only."""
import numpy as np
import pytest
import torch

import joiner_reference as jr
import lattice_reference as lr
import pruned_joiner_reference as pjr
import pruned_reference as pr

I32_MAX = 2 ** 31 - 1


def _inputs(seed, N=4, T=6, U=5, H=16, V=7, bias=True, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(N, T, H, generator=g).to(dtype)
    pred = torch.randn(N, U, H, generator=g).to(dtype)
    weight = (torch.randn(V, H, generator=g) / H ** 0.5).to(dtype)
    b = torch.randn(V, generator=g).to(dtype) if bias else None
    labels = torch.randint(0, V, (N, U - 1), generator=g, dtype=torch.int32)
    act_lens = torch.tensor([T] + [max(1, T - 1 - i) for i in range(N - 1)], dtype=torch.int32)
    label_lens = torch.tensor([U - 1] + [(i % U) for i in range(N - 1)], dtype=torch.int32)
    return enc, pred, weight, b, labels, act_lens, label_lens


def window(kind, seed, act_lens, label_lens, T, U, R):
    """[N, T] int32 window starts of one kind."""
    rng = np.random.default_rng(seed)
    N = act_lens.shape[0]
    if kind == "monotone":
        r = pr.random_monotone_ranges(rng, act_lens.numpy(), label_lens.numpy(), T, R)
    elif kind == "zero":
        r = np.zeros((N, T))
    elif kind == "negative":
        r = rng.integers(-R - 1, 1, (N, T))
    elif kind == "beyond":
        r = label_lens.numpy()[:, None] + rng.integers(-1, 3, (N, T))
    elif kind == "non_monotone":
        r = rng.integers(-2, U + 2, (N, T))
    elif kind == "extreme":
        r = rng.choice([-I32_MAX - 1, -I32_MAX, I32_MAX, I32_MAX - 1, 0, 1], (N, T))
    return torch.tensor(np.asarray(r, np.int64), dtype=torch.int32)


def pruned_hidden(enc, pred, ranges, R, activation):
    """[N, T, R, H] h of the rows prune_joint_inputs gives (clamped u on padding rows, as there)."""
    U = pred.shape[1]
    idx = (ranges.long()[..., None] + torch.arange(R)).clamp(0, U - 1)
    s = enc.float()[:, :, None, :] + pred.float()[torch.arange(enc.shape[0])[:, None, None], idx]
    a = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    return a.to(torch.bfloat16), idx


CASES = [("monotone", 2), ("monotone", 3), ("zero", 1), ("zero", 5), ("zero", 8), ("negative", 3), ("beyond", 2),
         ("non_monotone", 3), ("extreme", 2), ("non_monotone", 7)]


@pytest.mark.parametrize("kind,R", CASES)
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_equals_prune_joint_inputs_joiner_and_pruned_loss(kind, R, activation):
    """Costs and the four gradients of the pruned lattice loss: R = 1, R = U (5), R > U (7, 8) among the cases."""
    blank = 0 if R % 2 else 6
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(R * 11 + len(kind))
    N, T, H = enc.shape
    U = pred.shape[1]
    ranges = window(kind, R, act_lens, label_lens, T, U, R)

    # the eager recipe: prune_joint_inputs -> joiner -> pruned loss
    hp, idx = pruned_hidden(enc, pred, ranges, R, activation)
    z = jr.logits(hp, weight, bias)
    costs_ref, dz = pr.pruned_loss(z.numpy(), labels.numpy(), act_lens.numpy(), label_lens.numpy(),
                                   ranges.numpy(), blank)
    dz = torch.tensor(dz)
    ds = (dz @ weight.double()) * jr.act_grad(hp, activation)
    de_ref = ds.sum(2)
    dp_ref = torch.zeros(N, U, H, dtype=torch.float64)
    dp_ref.index_put_((torch.arange(N)[:, None, None].expand_as(idx), idx), ds, accumulate=True)
    dw_ref = torch.einsum('ntrv,ntrh->vh', dz, hp.double())
    db_ref = dz.sum((0, 1, 2))

    # the masked dense reference through the lattice loss
    h = jr.hidden(enc, pred, activation)
    px, py = pjr.log_probs(h, weight, bias, labels, act_lens, label_lens, ranges, R, blank)
    costs, gx, gy = lr.loss(px.numpy(), py.numpy(), act_lens.numpy(), label_lens.numpy())
    np.testing.assert_allclose(costs, costs_ref, rtol=1e-12, atol=1e-12)
    got = pjr.gradients(h, weight, bias, labels, act_lens, label_lens, torch.tensor(gx), torch.tensor(gy), ranges, R,
                        activation, blank)
    for g, r in zip(got, (de_ref, dp_ref, dw_ref, db_ref)):
        torch.testing.assert_close(g, r, rtol=1e-12, atol=1e-12)


def test_full_window_from_zero_is_the_dense_reference():
    enc, pred, weight, bias, labels, act_lens, label_lens = _inputs(3)
    N, T, _ = enc.shape
    U = pred.shape[1]
    h = jr.hidden(enc, pred, 'tanh')
    ranges = torch.zeros(N, T, dtype=torch.int32)
    for a, b in zip(pjr.log_probs(h, weight, bias, labels, act_lens, label_lens, ranges, U),
                    jr.log_probs(h, weight, bias, labels, act_lens, label_lens)):
        assert torch.equal(a, b)


def test_extreme_starts_cover_nothing_and_do_not_wrap():
    _, _, _, _, _, act_lens, label_lens = _inputs(1)
    ranges = torch.tensor([[I32_MAX, -I32_MAX - 1, I32_MAX - 1, -I32_MAX, 0, 0]] * 4, dtype=torch.int32)
    cov = pjr.covered(ranges, 3, act_lens, label_lens, 6, 5)
    assert not cov[:, :4].any()
    assert cov[0, 4, :3].all() and not cov[0, 4, 3:].any()


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_explicit_gradients_are_fp64_autograd(activation):
    enc, pred, weight, b, labels, act_lens, label_lens = _inputs(7, dtype=torch.float64)
    N, T, _ = enc.shape
    U = pred.shape[1]
    ranges = window("non_monotone", 4, act_lens, label_lens, T, U, 3)
    mx, my = pjr.factor_masks(ranges, 3, act_lens, label_lens, T, U)
    leaves = [t.clone().requires_grad_(True) for t in (enc, pred, weight, b)]
    px, py = jr.fp64_forward(*leaves, labels, act_lens, label_lens, activation, blank=2)
    g = torch.Generator().manual_seed(3)
    dpx = torch.randn(px.shape, generator=g, dtype=torch.float64)
    dpy = torch.randn(py.shape, generator=g, dtype=torch.float64)
    ((px.where(mx, torch.zeros_like(px)) * dpx).sum() + (py.where(my, torch.zeros_like(py)) * dpy).sum()).backward()
    dpx[~mx] = float('nan')   # off the covered cells: never read
    dpy[~my] = float('nan')
    s = enc[:, :, None, :] + pred[:, None, :, :]
    h = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    got = pjr.gradients(h, weight, b, labels, act_lens, label_lens, dpx, dpy, ranges, 3, activation, blank=2)
    for x, leaf in zip(got, leaves):
        torch.testing.assert_close(x, leaf.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_masked_fp64_form_passes_gradcheck(activation):
    enc, pred, weight, b, labels, act_lens, label_lens = _inputs(11, N=2, T=3, U=3, H=16, V=5, dtype=torch.float64)
    if activation == 'relu':   # keep every pre-activation away from the kink
        enc = enc + torch.sign(enc) * 0.1
    ranges = torch.tensor([[0, 1, -1], [1, 0, 2]], dtype=torch.int32)
    mx, my = pjr.factor_masks(ranges, 2, act_lens, label_lens, 3, 3)

    def f(e, p, w, bb):
        px, py = jr.fp64_forward(e, p, w, bb, labels, act_lens, label_lens, activation)
        return px[mx], py[my]

    args = [t.clone().requires_grad_(True) for t in (enc, pred, weight, b)]
    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-7)
