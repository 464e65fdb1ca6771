"""The fp64 delay-penalty reference (tests/delay_reference.py) against independent formulations, without a GPU."""
import numpy as np
import pytest
import torch

import delay_reference as dr
import pruned_reference as pr
import smoothed_reference as sr


def case(seed, N=3, T=4, U=3, V=5, full=False):
    rng = np.random.default_rng(seed)
    acts = rng.standard_normal((N, T, U, V))
    labels = rng.integers(1, V, size=(N, max(U - 1, 1))).astype(np.int32)
    act_lens = np.array([T] + [int(rng.integers(1, T + 1)) for _ in range(N - 1)], np.int32)
    label_lens = np.array([U - 1] + [int(rng.integers(0, U)) for _ in range(N - 1)], np.int32)
    if full:
        act_lens[:], label_lens[:] = T, U - 1
    return acts, labels, act_lens, label_lens


@pytest.mark.parametrize("lam", [0.0, 0.3, 2.0])
@pytest.mark.parametrize("T,U", [(1, 1), (1, 3), (4, 1), (2, 2), (3, 3), (4, 3), (4, 2)])
def test_brute_force_paths(T, U, lam):
    acts, labels, act_lens, label_lens = case(T * 10 + U, N=2, T=T, U=U, full=True)
    costs, _ = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam)
    for b in range(2):
        want = dr.brute_force(acts[b], labels[b], T, U, delay_penalty=lam)
        assert costs[b] == pytest.approx(want, rel=1e-12, abs=1e-12)


def test_penalty_favours_early_labels():
    """Two equally likely paths of one label: the earlier emission gains lambda per frame of lead."""
    T, U, V = 3, 2, 3
    acts = np.zeros((1, T, U, V))
    labels = np.array([[1]], np.int32)
    lens, ylens = np.array([T], np.int32), np.array([1], np.int32)
    c0 = dr.dense_loss(acts, labels, lens, ylens)[0][0]
    c1 = dr.dense_loss(acts, labels, lens, ylens, delay_penalty=1.0)[0][0]
    # uniform logits: every path has the same plain score; the penalties are 1, 0 and -1 for t = 0, 1, 2
    assert c1 - c0 == pytest.approx(-np.log(np.mean(np.exp([1.0, 0.0, -1.0]))), rel=1e-12)


def test_negative_cost_at_large_penalty():
    acts, labels, act_lens, label_lens = case(5, N=1, T=6, U=3, full=True)
    costs, grads = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=4.0)
    assert costs[0] < 0
    assert np.isfinite(grads).all()


class _DenseLoss(torch.autograd.Function):
    """The reference's cost with its own gradient, for torch.autograd.gradcheck."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, lam):
        c, g = dr.dense_loss(acts.detach().numpy(), labels, act_lens, label_lens, delay_penalty=lam)
        ctx.save_for_backward(torch.from_numpy(g))
        return torch.from_numpy(c)

    @staticmethod
    def backward(ctx, go):
        (g,) = ctx.saved_tensors
        return go[:, None, None, None] * g, None, None, None, None


@pytest.mark.parametrize("lam", [0.0, 0.7])
def test_gradcheck(lam):
    acts, labels, act_lens, label_lens = case(11, N=3, T=4, U=3, V=4)
    x = torch.tensor(acts, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a: _DenseLoss.apply(a, labels, act_lens, label_lens, lam), (x,),
                                    eps=1e-6, atol=1e-7, rtol=1e-5)


@pytest.mark.parametrize("lam", [0.0, 0.5])
def test_torch_lattice_matches(lam):
    """The torch fp64 form (autograd) and the numpy form agree on costs and gradients."""
    acts, labels, act_lens, label_lens = case(12, N=3, T=5, U=4, V=6)
    x = torch.tensor(acts, requires_grad=True)
    c = dr.torch_dense_costs(x, labels, act_lens, label_lens, delay_penalty=lam)
    c.sum().backward()
    want_c, want_g = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam)
    np.testing.assert_allclose(c.detach().numpy(), want_c, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(x.grad.numpy(), want_g, rtol=1e-10, atol=1e-12)


def test_zero_is_the_plain_reference():
    acts, labels, act_lens, label_lens = case(13, N=4, T=5, U=4, V=6)
    N, T, U, V = acts.shape
    c0, g0 = pr.pruned_loss(acts, labels, act_lens, label_lens, np.zeros((N, T), np.int32))
    c1, g1 = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=0.0)
    assert np.array_equal(c0, c1) and np.array_equal(g0, g1)
    rng = np.random.default_rng(1)
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    for lm, am in ((0.0, 0.0), (0.25, 0.0), (0.25, 0.1)):
        want = sr.reference(trans, pred, labels, act_lens, label_lens, lm, am)
        got = dr.joint_reference(trans, pred, labels, act_lens, label_lens, lm, am, delay_penalty=0.0)
        for w, g in zip(want, got):
            np.testing.assert_allclose(g, w, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("lam,fe", [(0.4, 0.0), (0.4, 0.3), (0.0, 0.3)])
def test_fastemit_surrogate(lam, fe):
    """gradient = d/dx [cost_penalised - fe sum sg[e_y] log p_y], e_y of the penalised lattice, p_y unpenalised."""
    acts, labels, act_lens, label_lens = case(14, N=3, T=5, U=4, V=6)
    _, g = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam, fastemit_lambda=fe)
    x = torch.tensor(acts, requires_grad=True)
    total = dr.torch_dense_costs(x, labels, act_lens, label_lens, delay_penalty=lam).sum()
    for b in range(acts.shape[0]):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        if U < 2:
            continue
        lp = pr.log_softmax(acts[b, :T, :U])
        y = labels[b, :U - 1].astype(np.int64)
        lpb = lp[:, :, 0]
        lpy = lp[:, np.arange(U - 1), y] + dr.penalty(T, U - 1, lam)
        alpha, beta, ll = pr.lattice(lpb, lpy)
        e_y = torch.tensor(np.exp(alpha[:, :U - 1] + lpy + beta[:, 1:] - ll))
        logp = torch.log_softmax(x[b, :T, :U - 1], dim=-1)[:, torch.arange(U - 1), torch.as_tensor(y)]
        total = total - fe * (e_y * logp).sum()
    total.backward()
    np.testing.assert_allclose(g, x.grad.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("lam", [0.0, 0.6])
def test_joint_reference(lm, am, lam):
    """The joint reference's costs equal the numpy factors'; unsmoothed, it is the dense reference on the
    materialised logits with the gradients summed onto the factors."""
    acts, labels, act_lens, label_lens = case(15, N=3, T=5, U=4, V=6)
    rng = np.random.default_rng(2)
    N, T, U, V = acts.shape
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    c, dF, dG = dr.joint_reference(trans, pred, labels, act_lens, label_lens, lm, am, delay_penalty=lam)
    np.testing.assert_allclose(c, dr.joint_costs(trans, pred, labels, act_lens, label_lens, lm, am, delay_penalty=lam),
                               rtol=1e-12, atol=1e-12)
    if lm == 0.0 and am == 0.0:
        cd, g = dr.dense_loss(trans[:, :, None] + pred[:, None], labels, act_lens, label_lens, delay_penalty=lam)
        np.testing.assert_allclose(c, cd, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(dF, g.sum(axis=2), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(dG, g.sum(axis=1), rtol=1e-10, atol=1e-12)


def test_pruned_reference_covered_cells():
    """Pruned: the penalty on the covered cells only; full windows give the dense loss."""
    acts, labels, act_lens, label_lens = case(16, N=3, T=5, U=4, V=6)
    N, T, U, V = acts.shape
    full = dr.loss(acts, labels, act_lens, label_lens, np.zeros((N, T), np.int32), delay_penalty=0.5)
    dense = dr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=0.5)
    for f, d in zip(full, dense):
        assert np.array_equal(f, d)
    R = 2
    rng = np.random.default_rng(3)
    ranges = pr.random_monotone_ranges(rng, act_lens, label_lens, T, R)
    logits = rng.standard_normal((N, T, R, V))
    c0, _ = pr.pruned_loss(logits, labels, act_lens, label_lens, ranges)
    c1, g1 = dr.loss(logits, labels, act_lens, label_lens, ranges, delay_penalty=0.0)
    assert np.array_equal(c0, c1)
    c2, g2 = dr.loss(logits, labels, act_lens, label_lens, ranges, delay_penalty=0.5)
    assert np.isfinite(g2).all() and not np.array_equal(c1, c2)
