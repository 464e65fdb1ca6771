"""The fp64 modified-topology reference (tests/modified_reference.py) against independent formulations, without a
GPU."""
import numpy as np
import pytest
import torch

import delay_reference as dr
import modified_reference as mr
import pruned_reference as pr
from test_delay_reference import case


@pytest.mark.parametrize("lam", [0.0, 0.4])
@pytest.mark.parametrize("T,U", [(1, 1), (1, 2), (2, 3), (4, 1), (2, 2), (3, 3), (4, 3), (5, 3), (5, 4), (3, 5)])
def test_brute_force_paths(T, U, lam):
    acts, labels, act_lens, label_lens = case(T * 10 + U, N=2, T=T, U=U, full=True)
    costs, grads = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam)
    for b in range(2):
        want = mr.brute_force(acts[b], labels[b], T, U, delay_penalty=lam)
        if np.isinf(want):
            assert U - 1 > T and costs[b] == np.inf
            assert not grads[b].any()
        else:
            assert costs[b] == pytest.approx(want, rel=1e-12, abs=1e-12)


def test_log_likelihoods_agree():
    """alpha's virtual cell and beta(0,0) are the same log-likelihood."""
    acts, labels, act_lens, label_lens = case(3, N=4, T=6, U=4, V=5)
    for b in range(4):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        lp = pr.log_softmax(acts[b, :T, :U])
        y = labels[b, :U - 1].astype(np.int64)
        alpha, beta, ll = mr.lattice(lp[:, :, 0], lp[:, np.arange(U - 1), y])
        assert beta[0, 0] == pytest.approx(ll, rel=1e-12, abs=1e-300) or (ll == beta[0, 0] == -np.inf)


class _DenseLoss(torch.autograd.Function):
    """The reference's cost with its own gradient, for torch.autograd.gradcheck."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, lam):
        c, g = mr.dense_loss(acts.detach().numpy(), labels, act_lens, label_lens, delay_penalty=lam)
        ctx.save_for_backward(torch.from_numpy(g))
        return torch.from_numpy(c)

    @staticmethod
    def backward(ctx, go):
        (g,) = ctx.saved_tensors
        return go[:, None, None, None] * g, None, None, None, None


@pytest.mark.parametrize("lam", [0.0, 0.7])
def test_gradcheck(lam):
    acts, labels, act_lens, label_lens = case(11, N=3, T=5, U=3, V=4, full=True)
    act_lens[1], label_lens[2] = 3, 1
    x = torch.tensor(acts, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a: _DenseLoss.apply(a, labels, act_lens, label_lens, lam), (x,),
                                    eps=1e-6, atol=1e-7, rtol=1e-5)


@pytest.mark.parametrize("lam", [0.0, 0.5])
def test_torch_lattice_matches(lam):
    """The torch fp64 form (autograd) and the numpy form agree on costs and gradients."""
    acts, labels, act_lens, label_lens = case(12, N=4, T=5, U=4, V=6)
    act_lens[3], label_lens[3] = 5, 3
    x = torch.tensor(acts, requires_grad=True)
    c = mr.torch_dense_costs(x, labels, act_lens, label_lens, delay_penalty=lam)
    c[torch.isfinite(c)].sum().backward()
    want_c, want_g = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam)
    np.testing.assert_allclose(c.detach().numpy(), want_c, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(x.grad.numpy(), want_g, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("lam", [0.0, 0.3])
def test_closed_forms(lam):
    """U_b = 1: every frame a blank, cost -sum_t lp_blank(t,0).  T_b = U_b - 1: every frame a label,
    cost -sum_t lp_y(t,t) (with the penalty)."""
    rng = np.random.default_rng(4)
    T, V = 5, 6
    acts = rng.standard_normal((2, T, T + 1, V))
    labels = rng.integers(1, V, size=(2, T)).astype(np.int32)
    act_lens = np.array([T, T], np.int32)
    label_lens = np.array([0, T], np.int32)
    costs, grads = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam)
    lp = pr.log_softmax(acts)
    assert costs[0] == pytest.approx(-lp[0, :, 0, 0].sum(), rel=1e-13)
    ts = np.arange(T)
    want = -(lp[1, ts, ts, labels[1]] + lam * ((T - 1) / 2.0 - ts)).sum()
    assert costs[1] == pytest.approx(want, rel=1e-13)
    # one path: occupancy 1 on it, the gradient is softmax - one_hot on the path's cells and zero elsewhere
    g = np.zeros_like(grads[1])
    for t in range(T):
        g[t, t] = np.exp(lp[1, t, t])
        g[t, t, labels[1, t]] -= 1.0
    np.testing.assert_allclose(grads[1], g, rtol=1e-12, atol=1e-13)


def test_no_path_is_inf_with_zero_gradient():
    rng = np.random.default_rng(5)
    acts = rng.standard_normal((3, 4, 6, 5))
    labels = rng.integers(1, 5, size=(3, 5)).astype(np.int32)
    act_lens = np.array([2, 4, 3], np.int32)
    label_lens = np.array([3, 5, 2], np.int32)     # U_b - 1 = 3 > 2, 5 > 4; 2 <= 3 has a path
    for lam, fe, clamp in ((0.0, 0.0, -1.0), (0.5, 0.3, 0.2)):
        costs, grads = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam, fastemit_lambda=fe,
                                     clamp=clamp)
        assert costs[0] == np.inf and costs[1] == np.inf and np.isfinite(costs[2])
        assert not grads[:2].any() and grads[2].any()
        assert mr.brute_force(acts[0], labels[0], 2, 4) == np.inf


@pytest.mark.parametrize("lam,fe", [(0.0, 0.3), (0.4, 0.3), (0.4, 0.0)])
def test_fastemit_surrogate(lam, fe):
    """gradient = d/dx [cost - fe sum sg[e_y] log p_y], e_y the modified (penalised) label occupancy, p_y unpenalised."""
    acts, labels, act_lens, label_lens = case(14, N=3, T=5, U=4, V=6)
    _, g = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=lam, fastemit_lambda=fe)
    x = torch.tensor(acts, requires_grad=True)
    total = mr.torch_dense_costs(x, labels, act_lens, label_lens, delay_penalty=lam).sum()
    for b in range(acts.shape[0]):
        T, U = int(act_lens[b]), int(label_lens[b]) + 1
        if U < 2:
            continue
        lp = pr.log_softmax(acts[b, :T, :U])
        y = labels[b, :U - 1].astype(np.int64)
        lpb = lp[:, :, 0]
        lpy = lp[:, np.arange(U - 1), y] + dr.penalty(T, U - 1, lam)
        alpha, beta, ll = mr.lattice(lpb, lpy)
        e_y = torch.tensor(mr.occupancies(alpha, beta, lpb, lpy, ll)[1])
        logp = torch.log_softmax(x[b, :T, :U - 1], dim=-1)[:, torch.arange(U - 1), torch.as_tensor(y)]
        total = total - fe * (e_y * logp).sum()
    total.backward()
    np.testing.assert_allclose(g, x.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_differs_from_regular():
    """The same logits score differently under the two topologies (a label also ends its frame here)."""
    acts, labels, act_lens, label_lens = case(6, N=3, T=5, U=3, V=5, full=True)
    cm, _ = mr.dense_loss(acts, labels, act_lens, label_lens)
    cr, _ = dr.dense_loss(acts, labels, act_lens, label_lens)
    assert not np.isclose(cm, cr, rtol=1e-6).any()


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("lam", [0.0, 0.6])
def test_joint_reference(lm, am, lam):
    """The joint reference's costs equal the numpy factors'; unsmoothed, it is the dense modified reference on the
    materialised logits with the gradients summed onto the factors.  One utterance has no path."""
    acts, labels, act_lens, label_lens = case(15, N=3, T=5, U=4, V=6)
    act_lens[2], label_lens[2] = 2, 3
    rng = np.random.default_rng(2)
    N, T, U, V = acts.shape
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    c, dF, dG = mr.joint_reference(trans, pred, labels, act_lens, label_lens, lm, am, delay_penalty=lam)
    np.testing.assert_allclose(c, mr.joint_costs(trans, pred, labels, act_lens, label_lens, lm, am, delay_penalty=lam),
                               rtol=1e-12, atol=1e-12)
    assert c[2] == np.inf and np.isfinite(dF).all() and np.isfinite(dG).all()
    assert not dF[2].any()
    if lm == 0.0 and am == 0.0:
        cd, g = mr.dense_loss(trans[:, :, None] + pred[:, None], labels, act_lens, label_lens, delay_penalty=lam)
        np.testing.assert_allclose(c, cd, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(dF, g.sum(axis=2), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(dG, g.sum(axis=1), rtol=1e-10, atol=1e-12)
        assert not dG[2].any()


def test_pruned_full_windows_and_adversarial_windows():
    """Full windows give the dense loss exactly; windows that leave no modified path give +inf and zeros."""
    acts, labels, act_lens, label_lens = case(16, N=3, T=5, U=4, V=6)
    N, T, U, V = acts.shape
    full = mr.loss(acts, labels, act_lens, label_lens, np.zeros((N, T), np.int32), delay_penalty=0.5)
    dense = mr.dense_loss(acts, labels, act_lens, label_lens, delay_penalty=0.5)
    for f, d in zip(full, dense):
        assert np.array_equal(f, d)
    # R = 3, T_b = 4, U_b = 4: windows that keep a modified path, then windows that advance 2 labels in frame 1 -
    # valid for the regular lattice, but a modified path is at u <= t on frame t, so it cannot reach them
    R = 3
    act_lens = np.array([4, 4, 4], np.int32)
    label_lens = np.array([3, 3, 3], np.int32)
    ranges = np.array([[0, 0, 1, 1, 1], [0, 1, 1, 1, 1], [0, 0, 0, 1, 1]], np.int32)
    rng = np.random.default_rng(3)
    logits = rng.standard_normal((N, T, R, V))
    costs, grads = mr.loss(logits, labels, act_lens, label_lens, ranges)
    assert np.isfinite(pr.pruned_loss(logits, labels, act_lens, label_lens, ranges)[0]).all()
    assert np.isfinite(costs).all()
    ranges_dead = np.array([[0, 2, 2, 2, 2]] * 3, np.int32)
    assert np.isfinite(pr.pruned_loss(logits, labels, act_lens, label_lens, ranges_dead)[0]).all()
    c2, g2 = mr.loss(logits, labels, act_lens, label_lens, ranges_dead)
    assert (c2 == np.inf).all() and not g2.any()


def test_ranges_from_modified_occupancies():
    """The modified ranges are pruned_reference's window rule on the modified occupancies; they keep the
    structural properties of include/rnnt.h."""
    acts, labels, act_lens, label_lens = case(17, N=4, T=8, U=5, V=7)
    act_lens[1], label_lens[1] = 2, 4          # no path: every frame scores 0, a = 0
    rng = np.random.default_rng(4)
    N, T, U, V = acts.shape
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    for R in (2, 3, 4):
        ranges, _ = mr.prune_ranges(trans, pred, labels, act_lens, label_lens, T, R)
        pr.check_range_properties(ranges, act_lens, label_lens, R)
        e_b, e_y = mr.joint_occupancies(trans, pred, labels, act_lens, label_lens)[0]
        T0 = int(act_lens[0])
        for t in range(1, T0 - 1):
            sc = pr.window_scores(e_b, e_y, t, R)
            assert sc.max() <= 1.0 + 1e-12
    # the utterance without a path scores every start 0 and takes a = 0 on every inner frame
    e_b, e_y = mr.joint_occupancies(trans, pred, labels, act_lens, label_lens)[1]
    assert not e_b.any() and not e_y.any()
