"""Pruned RNN-T loss and its pruning ranges on the GPU (DESIGN.md §8): bitwise identity with the dense loss,
the fp64 reference (tests/pruned_reference.py) for every streaming kernel, adversarial windows, the gradient
options, the ranges kernel, and the operators end to end through autograd."""
import ctypes as C

import numpy as np
import pytest
import torch

from pruned_reference import (check_range_properties, prune_ranges, pruned_loss, random_monotone_ranges,
                              simple_occupancies)

pytestmark = pytest.mark.gpu

# N, T, U, V, blank -> the streaming kernel that runs (fp32; fp64 rows are twice as long)
SHAPES = [
    (4, 9, 5, 5, 4),       # chunk, V odd, blank last
    (3, 10, 7, 50, 0),     # chunk, pairs
    (3, 6, 3, 257, 0),     # register tile, VEC 1
    (2, 5, 3, 502, 3),     # register tile, VEC 2
    (2, 4, 3, 1000, 7),    # register tile, VEC 4
    (2, 5, 3, 5002, 0),    # CTA per row, VEC 2
    (2, 4, 3, 1028, 5),    # CTA per row, VEC 4
    (4, 20, 33, 6, 0),     # multi-warp lattice
    (3, 40, 1, 6, 0),      # U == 1
    (3, 1, 5, 6, 0),       # T == 1
]
SID = lambda s: "N%d_T%d_U%d_V%d_b%d" % s   # noqa: E731
CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.float64: 3}
DTYPES = [torch.float32, torch.float64, torch.bfloat16, torch.float16]


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    import warprnnt_pytorch.pruned   # noqa: F401  (argtypes of the pruned entries)
    return wr


def make(seed, N, T, U, V, blank=0):
    rng = np.random.default_rng(seed)
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 1))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return rng, labels, tl, ul


def dev(*arrays):
    return tuple(torch.as_tensor(np.ascontiguousarray(a)).cuda() for a in arrays)


def dense_call(wr, acts, labels, tl, ul, blank, lam=0.0, clamp=0.0):
    N, T, U, V = acts.shape
    cdt = torch.float64 if acts.dtype == torch.float64 else torch.float32
    costs = torch.full((N,), float("nan"), dtype=cdt, device="cuda")
    grads = torch.full_like(acts, float("nan"))
    ws = torch.empty(wr.workspace_size(T, U, N, 8 if acts.dtype == torch.float64 else 4), dtype=torch.uint8,
                     device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=blank,
                         maxT=T, maxU=U, batch_first=True)
    st = wr.lib().rnnt_b200_loss_async_ex(CODE[acts.dtype], 0, acts.data_ptr(), grads.data_ptr(), labels.data_ptr(),
                                          ul.data_ptr(), tl.data_ptr(), V, N, costs.data_ptr(), 1.0,
                                          wr.rnntGradOptions(lam, clamp), ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    torch.cuda.synchronize()
    return costs, grads


def pruned_call(wr, logits, ranges, labels, tl, ul, U, blank, lam=0.0, clamp=0.0, scale=1.0):
    """rnnt_b200_pruned_loss_async_ex; logits [N,T,R,V], U the full lattice width."""
    from warprnnt_pytorch.pruned import pruned_workspace_size
    N, T, R, V = logits.shape
    cdt = torch.float64 if logits.dtype == torch.float64 else torch.float32
    costs = torch.full((N,), float("nan"), dtype=cdt, device="cuda")
    grads = torch.full_like(logits, float("nan"))
    ws = torch.empty(pruned_workspace_size(T, U, R, N, 8 if logits.dtype == torch.float64 else 4),
                     dtype=torch.uint8, device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=blank,
                         maxT=T, maxU=U, batch_first=True)
    st = wr.lib().rnnt_b200_pruned_loss_async_ex(CODE[logits.dtype], 0, logits.data_ptr(), grads.data_ptr(),
                                                 ranges.data_ptr(), R, labels.data_ptr(), ul.data_ptr(),
                                                 tl.data_ptr(), V, N, costs.data_ptr(), scale,
                                                 wr.rnntGradOptions(lam, clamp), ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    torch.cuda.synchronize()
    return costs, grads


# ---- 1. identity: R = U, ranges == 0 is the dense loss, bitwise --------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "fp64", "bf16", "fp16"])
@pytest.mark.parametrize("shape", SHAPES, ids=SID)
def test_identity_bitwise(wr, shape, dtype):
    N, T, U, V, blank = shape
    rng, labels_np, tl_np, ul_np = make(11, N, T, U, V, blank)
    acts = torch.tensor(rng.standard_normal((N, T, U, V)) * 3, dtype=dtype, device="cuda")
    labels, tl, ul = dev(labels_np, tl_np, ul_np)
    ranges = torch.zeros((N, T), dtype=torch.int32, device="cuda")
    for lam, clamp in ((0.0, 0.0), (0.5, 0.05)):
        c_d, g_d = dense_call(wr, acts, labels, tl, ul, blank, lam, clamp)
        c_p, g_p = pruned_call(wr, acts, ranges, labels, tl, ul, U, blank, lam, clamp)
        assert torch.equal(c_p, c_d)
        assert torch.equal(g_p, g_d)


def padding_mask(ranges, tl, ul, R):
    """[N, T, R] True where the row is padding (t >= T_b, u < 0, u >= U_b)."""
    N, T = ranges.shape
    u = ranges[:, :, None].astype(np.int64) + np.arange(R)
    t = np.arange(T)[None, :, None]
    return (t >= tl[:, None, None]) | (u < 0) | (u >= (ul + 1)[:, None, None])


def check_against_reference(wr, logits_np, ranges_np, labels_np, tl_np, ul_np, U, blank, dtype, lam=0.0, clamp=-1.0):
    logits = torch.tensor(logits_np, dtype=dtype, device="cuda")
    labels, tl, ul, ranges = dev(labels_np, tl_np, ul_np, ranges_np)
    c, g = pruned_call(wr, logits, ranges, labels, tl, ul, U, blank, lam, max(clamp, 0.0))
    c_ref, g_ref = pruned_loss(logits_np, labels_np, tl_np, ul_np, ranges_np, blank, lam, clamp)
    c, g = c.cpu().numpy(), g.cpu().numpy()
    assert not np.isnan(g).any()
    fin = np.isfinite(c_ref)
    assert (np.isinf(c) == ~fin).all(), (c, c_ref)
    assert np.allclose(c[fin], c_ref[fin], rtol=1e-5 if dtype == torch.float32 else 1e-11)
    assert (np.abs(g - g_ref) <= 1e-4 * np.abs(g_ref) + 1e-6).all(), np.abs(g - g_ref).max()
    R = logits_np.shape[2]
    assert not g[padding_mask(ranges_np, tl_np, ul_np, R)].any()      # padding rows: exact zeros
    assert not g[~fin].any()                                            # no path: all-zero gradient
    return c_ref


# ---- 2. reference: ranges from the reference algorithm, and random monotone ones ---------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("shape", SHAPES[:8], ids=SID)
@pytest.mark.parametrize("R", [2, 4])
def test_against_reference(wr, shape, dtype, R):
    N, T, U, V, blank = shape
    rng, labels_np, tl_np, ul_np = make(21, N, T, U, V, blank)
    logits = rng.standard_normal((N, T, R, V)) * 2
    D = 8
    trans, pred = rng.standard_normal((N, T, D)), rng.standard_normal((N, U, D))
    occ = simple_occupancies(trans, pred, labels_np % D, tl_np, ul_np, blank % D)
    from_alg, _ = prune_ranges(occ, T, R)
    for ranges in (from_alg, random_monotone_ranges(rng, tl_np, ul_np, T, R)):
        check_against_reference(wr, logits, ranges, labels_np[:, :U - 1], tl_np, ul_np, U, blank, dtype)


# ---- 3. adversarial windows ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("V", [6, 300, 2000])
def test_adversarial_ranges(wr, dtype, V):
    N, T, U, R, blank = 5, 8, 6, 3, 0
    rng, labels_np, tl_np, ul_np = make(31, N, T, U, V, blank)
    tl_np[:], ul_np[:] = T, U - 1
    logits = rng.standard_normal((N, T, R, V)) * 2
    ranges = random_monotone_ranges(rng, tl_np, ul_np, T, R)
    ranges[1] = rng.integers(-4, U + 4, size=T)                # anything, decreasing included
    ranges[2] = np.sort(ranges[2])[::-1]                       # decreasing: no path
    ranges[3] = [2 ** 31 - 1, -2 ** 31] * (T // 2)             # int32 extremes: every row padding
    ranges[4, :2] = [-1, -2]                                   # frame 0 reaches u = 0 only through s = 1
    c_ref = check_against_reference(wr, logits, ranges.astype(np.int32), labels_np[:, :U - 1], tl_np, ul_np, U,
                                    blank, dtype)
    assert np.isinf(c_ref[2]) and np.isinf(c_ref[3]) and np.isfinite(c_ref[0])


def test_infeasible_neighbours_unaffected(wr):
    """An utterance without a path leaves its neighbours bitwise as they are without it."""
    N, T, U, V, R = 4, 7, 6, 40, 2
    rng, labels_np, tl_np, ul_np = make(33, N, T, U, V)
    tl_np[:], ul_np[:] = T, U - 1
    logits = torch.tensor(rng.standard_normal((N, T, R, V)), dtype=torch.float32, device="cuda")
    ranges_np = random_monotone_ranges(rng, tl_np, ul_np, T, R)
    labels, tl, ul, ranges = dev(labels_np, tl_np, ul_np, ranges_np)
    c0, g0 = pruned_call(wr, logits, ranges, labels, tl, ul, U, 0)
    ranges_np[2] = 0
    c1, g1 = pruned_call(wr, logits, dev(ranges_np)[0], labels, tl, ul, U, 0)
    assert torch.isinf(c1[2]) and not g1[2].any()
    keep = [0, 1, 3]
    assert torch.equal(c0[keep], c1[keep]) and torch.equal(g0[keep], g1[keep])


# ---- 4. gradient options ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("shape", [SHAPES[1], SHAPES[3], SHAPES[5]], ids=SID)
def test_gradient_options(wr, shape, dtype):
    N, T, U, V, blank = shape
    R = 3
    rng, labels_np, tl_np, ul_np = make(41, N, T, U, V, blank)
    logits = rng.standard_normal((N, T, R, V)) * 3
    ranges = random_monotone_ranges(rng, tl_np, ul_np, T, R)
    lam = float(np.float32(0.5))
    _, g_fe = pruned_loss(logits, labels_np[:, :U - 1], tl_np, ul_np, ranges, blank, lam)
    nz = np.abs(g_fe[g_fe != 0])
    clamp = float(np.float32(np.quantile(nz, 0.97)))
    for c in (-1.0, clamp):
        check_against_reference(wr, logits, ranges, labels_np[:, :U - 1], tl_np, ul_np, U, blank, dtype, lam, c)


# ---- 5. the ranges kernel -----------------------------------------------------------------------------------------
def joint_ranges(trans, pred, labels, tl, ul, R, blank=0):
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    t, p = (torch.tensor(x, dtype=torch.float32, device="cuda") for x in (trans, pred))
    lab, tl_d, ul_d = dev(labels, tl, ul)
    _, ranges = add_joint_rnnt_loss_with_ranges(t, p, lab, tl_d, ul_d, R, blank, reduction='none')
    torch.cuda.synchronize()
    return ranges


def peaked_inputs(seed, N, T, U, V, R):
    """Factors scaled so that each frame's occupancy sits on a few cells and the best window beats the runner-up by
    more than 1e-4 on every frame: the most peaked scale (4, 2, 1) and seed that gives such a margin."""
    for scale in (4.0, 2.0, 1.0):
        for k in range(30):
            rng = np.random.default_rng(seed + 1000 * k)
            labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
            tl = np.full(N, T, np.int32)
            ul = rng.integers(U // 2, U, size=N).astype(np.int32)
            ul[0] = U - 1
            trans = rng.standard_normal((N, T, V)) * scale
            pred = rng.standard_normal((N, U, V)) * scale
            occ = simple_occupancies(trans, pred, labels, tl, ul)
            ranges, margin = prune_ranges(occ, T, R)
            if margin > 1e-4:
                return trans, pred, labels, tl, ul, ranges
    pytest.fail("no peaked input found")


@pytest.mark.parametrize("shape", [(3, 12, 8, 16, 3), (2, 20, 40, 24, 4), (2, 9, 5, 1030, 2)])
def test_ranges_kernel_equals_reference(wr, shape):
    N, T, U, V, R = shape
    trans, pred, labels, tl, ul, ref = peaked_inputs(5, N, T, U, V, R)
    got = joint_ranges(trans, pred, labels, tl, ul, R).cpu().numpy()
    assert np.array_equal(got, ref), (got, ref)


@pytest.mark.parametrize("R", [2, 3, 5, 64])
def test_ranges_kernel_properties(wr, R):
    rng = np.random.default_rng(R)
    N, T, U, V = 8, 30, 37, 33
    trans, pred = rng.standard_normal((N, T, V)), rng.standard_normal((N, U, V))
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(1, T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0], tl[1], ul[1] = T, U - 1, 1, 3
    first = joint_ranges(trans, pred, labels, tl, ul, R)
    check_range_properties(first.cpu().numpy(), tl, ul, R)
    assert torch.equal(first, joint_ranges(trans, pred, labels, tl, ul, R))   # deterministic


# ---- 6. end to end --------------------------------------------------------------------------------------------------
def torch_lattice_nll(lpb, lpy):
    """-log P of the lattice (lpb [T,U], lpy [T,U-1] tensors) by a log-sum-exp DP, differentiable."""
    T, U = lpb.shape
    prev = None
    for t in range(T):
        row = []
        for u in range(U):
            terms = []
            if t == 0 and u == 0:
                terms.append(torch.zeros((), dtype=lpb.dtype, device=lpb.device))
            if t > 0:
                terms.append(prev[u] + lpb[t - 1, u])
            if u > 0:
                terms.append(row[u - 1] + lpy[t, u - 1])
            terms = [x for x in terms if torch.isfinite(x)]   # all-dead cells: no NaN through logsumexp
            row.append(torch.logsumexp(torch.stack(terms), 0) if terms else
                       torch.tensor(-np.inf, dtype=lpb.dtype, device=lpb.device))
        prev = row
    return -(prev[U - 1] + lpb[T - 1, U - 1])


def torch_simple(trans, pred, labels, tl, ul, blank):
    out = []
    for b in range(trans.shape[0]):
        T, U = int(tl[b]), int(ul[b]) + 1
        lp = torch.log_softmax(trans[b, :T, None] + pred[b, None, :U], -1)
        lpy = lp[:, torch.arange(U - 1), torch.as_tensor(labels[b, :U - 1], dtype=torch.long)]
        out.append(torch_lattice_nll(lp[:, :, blank], lpy))
    return torch.stack(out)


def torch_pruned(logits, labels, tl, ul, ranges, blank):
    out = []
    ninf = torch.tensor(-np.inf, dtype=logits.dtype)
    for b in range(logits.shape[0]):
        T, U = int(tl[b]), int(ul[b]) + 1
        lp = torch.log_softmax(logits[b], -1)
        lpb = [[ninf] * U for _ in range(T)]
        lpy = [[ninf] * max(U - 1, 1) for _ in range(T)]
        for t in range(T):
            for s in range(logits.shape[2]):
                u = int(ranges[b, t]) + s
                if 0 <= u < U:
                    lpb[t][u] = lp[t, s, blank]
                    if u < U - 1:
                        lpy[t][u] = lp[t, s, int(labels[b, u])]
        lpb_t = torch.stack([torch.stack(r) for r in lpb])
        lpy_t = torch.stack([torch.stack(r) for r in lpy])
        out.append(torch_lattice_nll(lpb_t, lpy_t))
    return torch.stack(out)


class Model(torch.nn.Module):
    def __init__(self, D, V, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.am = torch.nn.Parameter(torch.randn(D, V, generator=g) * 0.5)
        self.lm = torch.nn.Parameter(torch.randn(D, V, generator=g) * 0.5)
        self.out = torch.nn.Parameter(torch.randn(D, V, generator=g) * 0.5)


def test_end_to_end_against_fp64_torch(wr):
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges, prune_joint_inputs, pruned_rnnt_loss
    N, T, U, D, V, R, blank = 3, 7, 5, 6, 9, 3, 0
    rng, labels_np, tl_np, ul_np = make(51, N, T, U, V, blank)
    enc_np, dec_np = rng.standard_normal((N, T, D)), rng.standard_normal((N, U, D))
    m32 = Model(D, V, 0).cuda()
    m64 = Model(D, V, 0).double()
    labels, tl, ul = dev(labels_np, tl_np, ul_np)
    enc = torch.tensor(enc_np, dtype=torch.float32, device="cuda", requires_grad=True)
    dec = torch.tensor(dec_np, dtype=torch.float32, device="cuda", requires_grad=True)
    simple, ranges = add_joint_rnnt_loss_with_ranges(enc @ m32.am, dec @ m32.lm, labels, tl, ul, R, blank,
                                                     reduction='sum')
    assert ranges.dtype == torch.int32 and ranges.shape == (N, T) and not ranges.requires_grad
    enc_p, dec_p = prune_joint_inputs(enc, dec, ranges, R)
    logits = torch.tanh(enc_p + dec_p) @ m32.out
    pruned = pruned_rnnt_loss(logits, labels, tl, ul, ranges, blank, reduction='sum')
    (0.5 * simple + pruned).backward()

    r = ranges.cpu().numpy()
    e64 = torch.tensor(enc_np, requires_grad=True)
    d64 = torch.tensor(dec_np, requires_grad=True)
    s64 = torch_simple(e64 @ m64.am, d64 @ m64.lm, labels_np, tl_np, ul_np, blank).sum()
    idx = torch.as_tensor(np.clip(r[:, :, None] + np.arange(R), 0, U - 1))
    dg = torch.gather(d64[:, None].expand(N, T, U, D), 2, idx[..., None].expand(N, T, R, D))
    lg64 = torch.tanh(e64[:, :, None] + dg) @ m64.out
    p64 = torch_pruned(lg64, labels_np, tl_np, ul_np, r, blank).sum()
    (0.5 * s64 + p64).backward()
    assert np.isclose(simple.item(), s64.item(), rtol=1e-5) and np.isclose(pruned.item(), p64.item(), rtol=1e-5)
    for a, b in ((enc.grad, e64.grad), (dec.grad, d64.grad), (m32.am.grad, m64.am.grad),
                 (m32.lm.grad, m64.lm.grad), (m32.out.grad, m64.out.grad)):
        a = a.double().cpu()
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (a - b).abs().max()


def test_full_window_equals_dense_operator(wr):
    """R = U through prune_joint_inputs: the pruned loss of the full joiner output is RNNTLoss of it."""
    from warprnnt_pytorch import RNNTLoss, prune_joint_inputs, pruned_rnnt_loss
    N, T, U, D, V = 3, 6, 4, 5, 30
    rng, labels_np, tl_np, ul_np = make(52, N, T, U, V)
    labels, tl, ul = dev(labels_np, tl_np, ul_np)
    enc = torch.tensor(rng.standard_normal((N, T, D)), dtype=torch.float32, device="cuda")
    dec = torch.tensor(rng.standard_normal((N, U, D)), dtype=torch.float32, device="cuda")
    W = torch.tensor(rng.standard_normal((D, V)), dtype=torch.float32, device="cuda")
    ranges = torch.zeros((N, T), dtype=torch.int32, device="cuda")
    enc_p, dec_p = prune_joint_inputs(enc, dec, ranges, U)
    lp = (torch.tanh(enc_p + dec_p) @ W).detach().requires_grad_()
    ld = (torch.tanh(enc[:, :, None] + dec[:, None]) @ W).detach().requires_grad_()
    assert torch.equal(lp, ld)
    a = pruned_rnnt_loss(lp, labels, tl, ul, ranges)
    b = RNNTLoss()(ld, labels, tl, ul)
    a.backward()
    b.backward()
    assert torch.equal(a, b) and torch.equal(lp.grad, ld.grad)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "fp64", "bf16", "fp16"])
def test_operator_reductions_and_grad_output(wr, dtype):
    from warprnnt_pytorch import PrunedRNNTLoss, pruned_rnnt_loss
    N, T, U, V, R = 4, 9, 6, 64, 3
    rng, labels_np, tl_np, ul_np = make(53, N, T, U, V)
    ranges_np = random_monotone_ranges(rng, tl_np, ul_np, T, R)
    labels, tl, ul, ranges = dev(labels_np[:, :U - 1], tl_np, ul_np, ranges_np)
    x = torch.tensor(rng.standard_normal((N, T, R, V)), dtype=dtype, device="cuda")
    wr_costs, wr_grads = pruned_call(wr, x, ranges, labels, tl, ul, U, 0)
    costs = {}
    for red in ('none', 'sum', 'mean'):
        xx = x.clone().requires_grad_()
        loss = PrunedRNNTLoss(reduction=red)(xx, labels, tl, ul, ranges)
        go = torch.arange(1, N + 1, dtype=loss.dtype, device="cuda") if red == 'none' else \
            torch.full_like(loss, 3.0)
        loss.backward(go)
        costs[red] = loss.detach()
        f = go[:, None, None, None] if red == 'none' else go * (1.0 / N if red == 'mean' else 1.0)
        want = (wr_grads.float() * f.float()).to(dtype)
        assert torch.allclose(xx.grad.float(), want.float(), rtol=1e-2 if dtype in (torch.bfloat16, torch.float16)
                              else 1e-6, atol=1e-6)
    assert torch.equal(costs['none'], wr_costs)
    assert torch.allclose(costs['sum'], wr_costs.sum().unsqueeze(0)) and \
        torch.allclose(costs['mean'], costs['sum'] / N)
    assert torch.equal(pruned_rnnt_loss(x, labels, tl, ul, ranges, reduction='none'), wr_costs)


def test_non_default_stream(wr):
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, V, R = 3, 8, 5, 100, 3
    rng, labels_np, tl_np, ul_np = make(54, N, T, U, V)
    ranges_np = random_monotone_ranges(rng, tl_np, ul_np, T, R)
    labels, tl, ul, ranges = dev(labels_np[:, :U - 1], tl_np, ul_np, ranges_np)
    x = torch.tensor(rng.standard_normal((N, T, R, V)), dtype=torch.float32, device="cuda")
    x0 = x.clone().requires_grad_()
    pruned_rnnt_loss(x0, labels, tl, ul, ranges, reduction='sum').backward()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x1 = x.clone().requires_grad_()
        loss = pruned_rnnt_loss(x1, labels, tl, ul, ranges, reduction='sum')
        loss.backward()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(x0.grad, x1.grad)


def test_operator_input_checks(wr):
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, V, R = 2, 4, 3, 8, 2
    x = torch.zeros((N, T, R, V), device="cuda")
    lab = torch.ones((N, U - 1), dtype=torch.int32, device="cuda")
    tl = torch.full((N,), T, dtype=torch.int32, device="cuda")
    ul = torch.full((N,), U - 1, dtype=torch.int32, device="cuda")
    rg = torch.zeros((N, T), dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError):
        pruned_rnnt_loss(x, lab, tl, ul, rg.long())
    with pytest.raises(ValueError):
        pruned_rnnt_loss(x, lab, tl, ul, rg[:, :T - 1].contiguous())
    with pytest.raises(ValueError):
        pruned_rnnt_loss(x, lab, tl, ul, torch.zeros((T, N), dtype=torch.int32, device="cuda").t())
    with pytest.raises(RuntimeError):
        pruned_rnnt_loss(x, lab, tl, ul, rg.cpu())
    with pytest.raises(ValueError):
        pruned_rnnt_loss(x, lab, tl + 1, ul, rg)     # T != max(act_lens)
