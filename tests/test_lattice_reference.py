"""The fp64 factor-level reference (tests/lattice_reference.py) against path enumeration, autograd, the dense logit
references, the constrained transducer's definition, and its no-path and unnormalised cases.  CPU only."""
import numpy as np
import pytest

import lattice_reference as lr
import modified_reference as mr
import pruned_reference as pr

TOPOLOGIES = [False, True]


def _random(rng, N, S, T, scale=1.0):
    return rng.standard_normal((N, S, T)) * scale, rng.standard_normal((N, S + 1, T)) * scale


@pytest.mark.parametrize("modified", TOPOLOGIES)
@pytest.mark.parametrize("T,U", [(1, 1), (1, 2), (3, 1), (3, 3), (4, 3), (5, 4), (2, 4), (6, 2)])
def test_against_path_enumeration(modified, T, U):
    rng = np.random.default_rng(T * 10 + U + 100 * modified)
    px, py = _random(rng, 1, U - 1, T, scale=2.0)
    costs, _, _ = lr.loss(px, py, [T], [U - 1], modified)
    lpb, lpy = lr.utterance_factors(px[0], py[0], T, U)
    bf = lr.brute_force(lpb, lpy, modified)
    if bf == np.inf:
        assert costs[0] == np.inf
    else:
        assert costs[0] == pytest.approx(bf, rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("modified", TOPOLOGIES)
@pytest.mark.parametrize("T,U", [(1, 1), (3, 2), (4, 4), (5, 3)])
def test_gradient_is_autograd_and_gradcheck(modified, T, U):
    import torch
    rng = np.random.default_rng(3 + T + 7 * U + modified)
    px, py = _random(rng, 1, U - 1, T)
    _, gx, gy = lr.loss(px, py, [T], [U - 1], modified)
    lpb = torch.tensor(py[0].T, requires_grad=True)
    lpy = torch.tensor(px[0].T, requires_grad=True)
    ll = lr.torch_ll(lpb, lpy, modified)
    ll_b, ll_y = torch.autograd.grad(ll, (lpb, lpy), allow_unused=True)
    ll_y = torch.zeros_like(lpy) if ll_y is None else ll_y
    np.testing.assert_allclose(gy[0], -ll_b.numpy().T, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gx[0], -ll_y.numpy().T, rtol=1e-10, atol=1e-12)
    assert torch.autograd.gradcheck(lambda b, y: lr.torch_ll(b, y, modified), (lpb, lpy))


def _dense_reference(logits, labels, act_lens, label_lens, modified):
    if modified:
        return mr.dense_loss(logits, labels, act_lens, label_lens)
    N, T, U, _ = logits.shape
    return pr.pruned_loss(logits, labels, act_lens, label_lens, np.zeros((N, T), np.int64))


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_log_softmax_factors_are_the_dense_loss(modified):
    """px / py gathered from log_softmax(logits): the costs are the dense loss's, and the chain rule through the
    gather gives its logit gradient."""
    rng = np.random.default_rng(11 + modified)
    N, T, U, V = 4, 7, 4, 6
    logits = rng.standard_normal((N, T, U, V))
    labels = rng.integers(1, V, (N, U - 1)).astype(np.int32)
    act_lens = np.array([7, 5, 3, 7], np.int32)
    label_lens = np.array([3, 2, 0, 1], np.int32)
    px, py = lr.factors_from_logits(logits, labels)
    costs, gx, gy = lr.loss(px, py, act_lens, label_lens, modified)
    ref_costs, ref_grad = _dense_reference(logits, labels, act_lens, label_lens, modified)
    np.testing.assert_allclose(costs, ref_costs, rtol=1e-12)
    p = np.exp(pr.log_softmax(logits))
    g = gy.transpose(0, 2, 1)[..., None] * -p
    g[..., 0] += gy.transpose(0, 2, 1)
    g[:, :, :U - 1] += gx.transpose(0, 2, 1)[..., None] * -p[:, :, :U - 1]
    for b in range(N):
        for u in range(U - 1):
            g[b, :, u, labels[b, u]] += gx[b, u]
    np.testing.assert_allclose(g, ref_grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("T,U", [(1, 1), (2, 2), (3, 3), (4, 2), (5, 4), (2, 4)])
def test_constrained_recipe(T, U):
    """k2's constrained transducer = the modified recursion on px + py[:, 1:, :]."""
    rng = np.random.default_rng(T + 13 * U)
    px, py = _random(rng, 1, U - 1, T, scale=1.5)
    costs, _, _ = lr.loss(px + py[:, 1:, :], py, [T], [U - 1], modified=True)
    lpb, lpy = lr.utterance_factors(px[0], py[0], T, U)
    bf = lr.constrained_brute_force(lpb, lpy)
    if bf == np.inf:
        assert costs[0] == np.inf
    else:
        assert costs[0] == pytest.approx(bf, rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_no_path_costs_inf_with_zero_gradient(modified):
    rng = np.random.default_rng(5)
    px, py = _random(rng, 3, 4, 6)
    px[0] = -np.inf                 # no label can be emitted: no path with labels
    py[1, :, :] = -np.inf           # no blank at all
    act_lens = np.array([6, 6, 3], np.int32)
    label_lens = np.array([4, 4, 4], np.int32)   # modified: more labels than frames
    if not modified:
        px[2, 1] = -np.inf          # label 1 can never be emitted
    costs, gx, gy = lr.loss(px, py, act_lens, label_lens, modified)
    assert (costs == np.inf).all()
    assert not gx.any() and not gy.any()


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_unnormalised_positive_factors(modified):
    rng = np.random.default_rng(17)
    px, py = _random(rng, 1, 3, 5)
    px, py = np.abs(px) + 2.0, np.abs(py) + 2.0
    costs, _, _ = lr.loss(px, py, [5], [3], modified)
    lpb, lpy = lr.utterance_factors(px[0], py[0], 5, 4)
    assert costs[0] < 0
    assert costs[0] == pytest.approx(lr.brute_force(lpb, lpy, modified), rel=1e-12)


def test_plus_inf_reads_as_nan():
    rng = np.random.default_rng(23)
    px, py = _random(rng, 2, 2, 4)
    py[0, 1, 2] = np.inf
    costs, _, _ = lr.loss(px, py, [4, 4], [2, 2])
    assert np.isnan(costs[0]) and np.isfinite(costs[1])
