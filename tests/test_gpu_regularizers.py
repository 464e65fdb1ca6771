"""Gradient options (FastEmit, clamp) on the GPU against the fp64 reference (tests/regularized_reference.py),
through every gradient kernel, storage type, layout, entry point and operator."""
import ctypes as C

import numpy as np
import pytest
import torch

from regularized_reference import rnnt_logits_reg

pytestmark = pytest.mark.gpu

# N, T, U, V, blank  -> the gradient kernel that runs (fp32; fp64 rows are twice as long)
SHAPES = [
    (4, 9, 5, 5, 4),       # chunk, V odd, blank last
    (3, 10, 7, 50, 0),     # chunk, pairs
    (2, 8, 5, 64, 1),      # chunk (fp64: 512 B rows, still chunk)
    (3, 6, 3, 257, 0),     # register tile, VEC 1
    (2, 5, 3, 502, 3),     # register tile, VEC 2
    (2, 4, 3, 1000, 7),    # register tile, VEC 4
    (2, 5, 3, 5002, 0),    # CTA per row, VEC 2
    (2, 4, 3, 1028, 5),    # CTA per row, VEC 4
    (1, 2, 2, 33001, 7),   # CTA per row, VEC 1, 17 trips
    (4, 20, 33, 6, 0),     # multi-warp lattice
    (3, 40, 1, 6, 0),      # U == 1
    (3, 1, 5, 6, 0),       # T == 1
]
# rnntGradOptions carries float32: the reference takes the options as the kernels see them (an fp64 gradient
# resolves the rounding of 0.01 or of a clamp to float32)
LAMBDAS = [float(np.float32(0.01)), 0.5]
CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.float64: 3}


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


def make_inputs(seed, N, T, U, V, blank=0):
    rng = np.random.default_rng(seed)
    acts = (rng.standard_normal((N, T, U, V)) * 3).astype(np.float32)
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return acts, labels, tl, ul


def to_dev(labels, tl, ul):
    N = len(tl)
    lab = labels if labels.size else np.zeros((N, 1), np.int32)
    return tuple(torch.as_tensor(np.ascontiguousarray(x)).cuda() for x in (lab, tl, ul))


def clip_for(g, tl, ul, frac=0.97):
    """A clamp that clips a few percent of the valid gradient elements."""
    valid = np.concatenate([g[b, :tl[b], :ul[b] + 1].reshape(-1) for b in range(g.shape[0])])
    return float(np.float32(np.quantile(np.abs(valid), frac))), valid


def loss_ex(wr, acts, labels, tl, ul, blank, lam, clamp, layout=0, scale=1.0):
    """rnnt_b200_loss_async_ex on device tensors; acts [N,T,U,V] (NTUV) or [T,U,N,V] (TUNV)."""
    N = tl.numel()
    T, U = (acts.shape[1], acts.shape[2]) if layout == 0 else (acts.shape[0], acts.shape[1])
    V = acts.shape[3]
    cdt = torch.float64 if acts.dtype == torch.float64 else torch.float32
    costs = torch.full((N,), float("nan"), dtype=cdt, device="cuda")
    grads = torch.full_like(acts, float("nan"))
    ws = torch.empty(wr.workspace_size(T, U, N, 8 if acts.dtype == torch.float64 else 4), dtype=torch.uint8,
                     device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=blank,
                         maxT=T, maxU=U, batch_first=True)
    st = wr.lib().rnnt_b200_loss_async_ex(CODE[acts.dtype], layout, acts.data_ptr(), grads.data_ptr(),
                                          labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N, costs.data_ptr(),
                                          scale, wr.rnntGradOptions(lam, clamp), ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    torch.cuda.synchronize()
    return costs, grads


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "N%d_T%d_U%d_V%d_b%d" % s)
def test_against_reference(wr, shape, dtype):
    N, T, U, V, blank = shape
    acts_np, labels_np, tl_np, ul_np = make_inputs(41, N, T, U, V, blank)
    acts = torch.tensor(acts_np, dtype=dtype, device="cuda")
    labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
    c_plain, g_plain = loss_ex(wr, acts, labels, tl, ul, blank, 0.0, 0.0)
    rtol, atol = (1e-4, 1e-6) if dtype == torch.float32 else (1e-8, 1e-12)
    for lam in LAMBDAS:
        c_ref, g_fe = rnnt_logits_reg(acts_np, labels_np, tl_np, ul_np, blank, fastemit_lambda=lam)
        clip, valid = clip_for(g_fe, tl_np, ul_np)
        assert (np.abs(valid) > clip).mean() >= 0.01
        for clamp in (-1.0, clip):
            g_ref = np.clip(g_fe, -clamp, clamp) if clamp > 0 else g_fe
            costs, g = loss_ex(wr, acts, labels, tl, ul, blank, lam, clamp)
            assert torch.equal(costs, c_plain)                       # the lattice and costs do not change
            g = g.cpu().numpy()
            assert np.allclose(costs.cpu().numpy(), c_ref, rtol=1e-5 if dtype == torch.float32 else 1e-11)
            bad = ~np.isclose(g, g_ref, rtol=rtol, atol=atol)
            assert not bad.any(), (lam, clamp, int(bad.sum()), np.abs(g - g_ref).max())
            for b in range(N):                                       # padded cells exact zeros
                assert not g[b, tl_np[b]:].any() and not g[b, :, ul_np[b] + 1:].any()
    assert not torch.equal(g_plain, torch.as_tensor(g).cuda()) or U == 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_sixteen_bit_storage(wr, dtype):
    """fp32 arithmetic inside: against the reference on the rounded inputs, the tolerance of the plain
    16-bit test (output rounding)."""
    from warprnnt_pytorch import RNNTLoss
    eps = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    for (N, T, U, V) in [(3, 11, 5, 64), (2, 7, 4, 5000), (2, 6, 3, 37), (2, 9, 34, 16), (1, 4, 2, 5001)]:
        acts_np, labels_np, tl_np, ul_np = make_inputs(43, N, T, U, V)
        acts_t = torch.tensor(acts_np).to(dtype)
        acts_np = acts_t.float().numpy().astype(np.float64)
        labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
        acts = acts_t.cuda()
        c_plain = torch.empty(N, device="cuda")
        wr.gpu_rnnt_async(acts, labels, tl, ul, c_plain, torch.empty_like(acts), 0)
        for lam in LAMBDAS:
            _, g_fe = rnnt_logits_reg(acts_np, labels_np, tl_np, ul_np, 0, fastemit_lambda=lam)
            clip, _ = clip_for(g_fe, tl_np, ul_np)
            for clamp in (-1.0, clip):
                g_ref = np.clip(g_fe, -clamp, clamp) if clamp > 0 else g_fe
                a = acts.clone().requires_grad_(True)
                out = RNNTLoss(reduction='none', fastemit_lambda=lam, clamp=clamp)(a, labels, tl, ul)
                out.sum().backward()
                assert torch.equal(out.detach(), c_plain)
                g = a.grad.float().cpu().numpy()
                assert np.allclose(g, g_ref, rtol=2 * eps, atol=1e-6), (N, T, U, V, lam, clamp, np.abs(g - g_ref).max())
                c2, g2 = torch.empty(N, device="cuda"), torch.empty_like(acts)   # the full entry, same kernels
                wr.gpu_rnnt_async(acts, labels, tl, ul, c2, g2, 0, fastemit_lambda=lam, clamp=clamp)
                torch.cuda.synchronize()
                assert torch.equal(c2, c_plain) and torch.equal(g2, a.grad)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_time_major_layout_is_the_transpose(wr, dtype):
    for (N, T, U, V, blank) in [(3, 10, 7, 50, 0), (2, 4, 3, 1000, 7), (2, 5, 3, 5002, 0)]:
        acts_np, labels_np, tl_np, ul_np = make_inputs(47, N, T, U, V, blank)
        acts = torch.tensor(acts_np, dtype=dtype, device="cuda")
        labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
        c0, g0 = loss_ex(wr, acts, labels, tl, ul, blank, 0.3, 0.02)
        c1, g1 = loss_ex(wr, acts.permute(1, 2, 0, 3).contiguous(), labels, tl, ul, blank, 0.3, 0.02, layout=1)
        assert torch.equal(c0, c1) and torch.equal(g1.permute(2, 0, 1, 3), g0)
        c2 = torch.empty_like(c0)
        g2 = torch.empty_like(g1)
        wr.gpu_rnnt_async_tunv(acts.permute(1, 2, 0, 3).contiguous(), labels, tl, ul, c2, g2, blank,
                               fastemit_lambda=0.3, clamp=0.02)
        torch.cuda.synchronize()
        assert torch.equal(c2, c0) and torch.equal(g2, g1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16, torch.float16],
                         ids=["fp32", "fp64", "bf16", "fp16"])
def test_ex_entries_without_options_equal_the_plain_entries(wr, dtype):
    for (N, T, U, V, blank) in [(3, 10, 7, 50, 0), (2, 6, 3, 257, 0), (2, 4, 3, 1028, 5)]:
        acts_np, labels_np, tl_np, ul_np = make_inputs(53, N, T, U, V, blank)
        acts = torch.tensor(acts_np, device="cuda").to(dtype)
        labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
        cdt = torch.float64 if dtype == torch.float64 else torch.float32
        c_plain, g_plain = torch.empty(N, dtype=cdt, device="cuda"), torch.empty_like(acts)
        wr.gpu_rnnt_async(acts, labels, tl, ul, c_plain, g_plain, blank, 0.5)
        torch.cuda.synchronize()
        c_ex, g_ex = loss_ex(wr, acts, labels, tl, ul, blank, 0.0, 0.0, scale=0.5)
        assert torch.equal(c_ex, c_plain) and torch.equal(g_ex, g_plain)
        if dtype in (torch.float32, torch.float64):
            c_tm, g_tm = torch.empty_like(c_plain), torch.empty_like(acts.permute(1, 2, 0, 3).contiguous())
            wr.gpu_rnnt_async_tunv(acts.permute(1, 2, 0, 3).contiguous(), labels, tl, ul, c_tm, g_tm, blank, 0.5)
            torch.cuda.synchronize()
            c_ex, g_ex = loss_ex(wr, acts.permute(1, 2, 0, 3).contiguous(), labels, tl, ul, blank, 0.0, 0.0,
                                 layout=1, scale=0.5)
            assert torch.equal(c_ex, c_tm) and torch.equal(g_ex, g_tm)
        # split backward: rnnt_b200_backward(_fp64/_16) against rnnt_b200_backward_ex with {0, 0}
        costs = torch.empty(N, dtype=cdt, device="cuda")
        ws = wr.gpu_rnnt_forward(acts, labels, tl, ul, costs, blank)
        w = torch.linspace(-1.0, 2.0, N, dtype=cdt, device="cuda")
        g_b = torch.full_like(acts, float("nan"))
        wr.gpu_rnnt_backward(acts, labels, tl, ul, g_b, w, blank, 0.25, ws)
        g_bx = torch.full_like(acts, float("nan"))
        opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream,
                             blank_label=blank, maxT=T, maxU=U, batch_first=True)
        st = wr.lib().rnnt_b200_backward_ex(CODE[dtype], acts.data_ptr(), g_bx.data_ptr(), labels.data_ptr(),
                                            ul.data_ptr(), tl.data_ptr(), V, N, w.data_ptr(), 0.25,
                                            wr.rnntGradOptions(0.0, 0.0), ws.data_ptr(), opt)
        assert st == 0
        torch.cuda.synchronize()
        assert torch.equal(g_b, g_bx)


def test_scale_and_upstream_gradient_fold_outside_the_clip():
    """out = grad_scale * grad_costs[b] * clip(g), through autograd for every reduction."""
    from warprnnt_pytorch import RNNTLoss
    N, T, U, V, blank = 5, 12, 6, 28, 0
    acts_np, labels_np, tl_np, ul_np = make_inputs(59, N, T, U, V, blank)
    labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
    lam = 0.3
    _, g_fe = rnnt_logits_reg(acts_np, labels_np, tl_np, ul_np, blank, fastemit_lambda=lam)
    clip, _ = clip_for(g_fe, tl_np, ul_np, 0.9)
    g_ref = np.clip(g_fe, -clip, clip)
    w = torch.tensor([1.0, -2.0, 0.5, 3.0, 0.0], device="cuda")
    for reduction, weight, factor in (('none', w, w.cpu().numpy()), ('sum', None, np.ones(N)),
                                      ('mean', None, np.full(N, 1.0 / N)), ('mean', 4.0, np.full(N, 4.0 / N))):
        acts = torch.tensor(acts_np, device="cuda", requires_grad=True)
        out = RNNTLoss(blank=blank, reduction=reduction, fastemit_lambda=lam, clamp=clip)(acts, labels, tl, ul)
        (out * weight).sum().backward() if weight is not None else out.sum().backward()
        want = g_ref * factor[:, None, None, None]
        assert np.allclose(acts.grad.cpu().numpy(), want, rtol=1e-4, atol=1e-6), reduction


def test_grouped_schedule_matches_the_split_backward(wr):
    """N = 16, T = 1500, U = 301, V = 50: the full call overlaps 4 batch groups (lattice of one group next to
    the streaming passes of the others); the split backward never groups.  Same per-row arithmetic."""
    N, T, U, V = 16, 1500, 301, 50
    rng = np.random.default_rng(61)
    acts = torch.randn(N, T, U, V, device="cuda", generator=torch.Generator("cuda").manual_seed(61))
    labels_np = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl_np = rng.integers(T // 2, T + 1, size=N).astype(np.int32)
    ul_np = rng.integers(U // 2, U, size=N).astype(np.int32)
    tl_np[0], ul_np[0] = T, U - 1
    labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
    lam, clamp = 0.01, 0.05
    c_full, g_full = loss_ex(wr, acts, labels, tl, ul, 0, lam, clamp)
    assert wr.last_launch_count() > 3                     # grouped: more than the three in-order launches
    costs = torch.empty(N, device="cuda")
    ws = wr.gpu_rnnt_forward(acts, labels, tl, ul, costs, 0)
    g_split = torch.full_like(acts, float("nan"))
    wr.gpu_rnnt_backward(acts, labels, tl, ul, g_split, None, 0, 1.0, ws, fastemit_lambda=lam, clamp=clamp)
    torch.cuda.synchronize()
    assert torch.equal(costs, c_full) and torch.equal(g_split, g_full)
    for b in (0, 5):
        Tb, Ub = int(tl_np[b]), int(ul_np[b]) + 1
        x = acts[b:b + 1, :Tb, :Ub].double().cpu().numpy()
        c_ref, g_ref = rnnt_logits_reg(x, labels_np[b:b + 1, :Ub - 1], [Tb], [Ub - 1], 0, fastemit_lambda=lam,
                                       clamp=clamp)
        assert np.allclose(c_full[b].item(), c_ref[0], rtol=1e-5)
        g = g_full[b, :Tb, :Ub].cpu().numpy()
        assert np.allclose(g, g_ref[0], rtol=1e-4, atol=1e-6), np.abs(g - g_ref[0]).max()
        del x, g_ref


def test_additive_joint_fastemit_matches_the_dense_operator():
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    for (N, T, U, V) in [(4, 20, 7, 64), (2, 33, 32, 130), (2, 6, 3, 5000)]:
        rng = np.random.default_rng(67)
        trans = torch.tensor(rng.standard_normal((N, T, V)).astype(np.float32), device="cuda", requires_grad=True)
        pred = torch.tensor(rng.standard_normal((N, U, V)).astype(np.float32), device="cuda", requires_grad=True)
        labels = torch.as_tensor(rng.integers(1, V, size=(N, U - 1)).astype(np.int32)).cuda()
        tl = torch.as_tensor(rng.integers(T // 2, T + 1, size=N).astype(np.int32)).cuda()
        ul = torch.as_tensor(rng.integers(0, U, size=N).astype(np.int32)).cuda()
        tl[0], ul[0] = T, U - 1
        w = torch.linspace(0.5, 1.5, N, device="cuda")
        out = AddJointRNNTLoss(reduction='none', fastemit_lambda=0.3)(trans, pred, labels, tl, ul)
        (out * w).sum().backward()
        g1, g2 = trans.grad.clone(), pred.grad.clone()
        trans.grad = pred.grad = None
        dense = RNNTLoss(reduction='none', fastemit_lambda=0.3)((trans.unsqueeze(2) + pred.unsqueeze(1)).contiguous(),
                                                               labels, tl, ul)
        (dense * w).sum().backward()
        assert torch.allclose(out, dense, rtol=1e-5, atol=1e-5)
        assert torch.allclose(g1, trans.grad, rtol=1e-4, atol=2e-6), (g1 - trans.grad).abs().max()
        assert torch.allclose(g2, pred.grad, rtol=1e-4, atol=2e-6), (g2 - pred.grad).abs().max()
        plain = AddJointRNNTLoss(reduction='none')(trans.detach(), pred.detach(), labels, tl, ul)
        assert torch.equal(plain, out.detach())


def test_sharded_loss_carries_the_options():
    """One process (no process group): ShardedRNNTLoss == RNNTLoss with the same options."""
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.distributed import ShardedRNNTLoss
    acts_np, labels_np, tl_np, ul_np = make_inputs(71, 4, 9, 5, 40)
    labels, tl, ul = to_dev(labels_np, tl_np, ul_np)
    grads = []
    for mod in (ShardedRNNTLoss(reduction='mean', fastemit_lambda=0.2, clamp=0.01),
                RNNTLoss(reduction='mean', fastemit_lambda=0.2, clamp=0.01)):
        acts = torch.tensor(acts_np, device="cuda", requires_grad=True)
        mod(acts, labels, tl, ul).sum().backward()
        grads.append(acts.grad)
    assert torch.allclose(grads[0], grads[1], rtol=1e-6, atol=0)
    _, g_fe = rnnt_logits_reg(acts_np, labels_np, tl_np, ul_np, 0, fastemit_lambda=0.2, clamp=0.01)
    assert np.allclose(grads[0].cpu().numpy(), g_fe / 4, rtol=1e-4, atol=1e-6)
