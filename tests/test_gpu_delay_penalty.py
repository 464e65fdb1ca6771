"""The delay penalty (DESIGN.md §10) on the GPU against the fp64 reference (tests/delay_reference.py).

Bars (§6): costs 1e-5 relative, gradients 1e-4 relative + 1e-6 absolute.  A penalised cost can cross zero, so the
cost bar is 1e-5 * max(|cost|, 1 + lambda T_b U_b / 2).  fp64 uses 1e-11 on costs and 1e-9 relative on gradients;
16-bit storage is compared with the reference on the rounded logits, gradients to the storage type's rounding."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import delay_reference as dr
import pruned_reference as pr
from joint_reference import grad_mismatch
from test_gpu_tuning_hooks import norm

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TORCH = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16, "fp16": torch.float16}
# (N, T, U, V): the dispatch family each shape reaches for fp32 (16-bit rows are half as long)
SHAPES = {
    "chunk": (4, 12, 6, 28),          # rows <= 512 B: rowstats / grad_chunk_kernel
    "tile": (3, 10, 5, 500),          # V / 4 <= 256 vectors: register tiles
    "row": (2, 6, 4, 1500),           # one CTA per row
    "wavefront_U65": (2, 30, 65, 20),     # multi-warp fp32 wavefront
    "wavefront_U301": (2, 8, 301, 12),
}
STORAGES = ["fp32", "fp64", "bf16", "fp16"]


def make(seed, N, T, U, V, blank=0):
    rng = np.random.default_rng(seed)
    acts = (rng.standard_normal((N, T, U, V)) * 1.5).astype(np.float32)
    labels = rng.integers(1, V, size=(N, max(U - 1, 1))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return acts, labels, tl, ul


def cuda(*xs):
    return [torch.as_tensor(x).cuda() for x in xs]


def f32(x):
    """The options reach the kernels as float32 (include/rnnt.h), fp64 calls included: the reference gets the same."""
    return float(np.float32(x))


def cost_bar(ref, lam, tl, ul, rel):
    return rel * np.maximum(np.abs(ref), 1.0 + lam * tl * (ul + 1) / 2.0)


def grad_tol(storage):
    return {"fp32": (1e-4, 1e-6), "fp64": (1e-9, 1e-12), "bf16": (1e-2, 1e-4), "fp16": (2e-3, 2e-5)}[storage]


def assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage):
    rel_c = 1e-11 if storage == "fp64" else 1e-5
    err = np.abs(costs - c_ref)
    bar = cost_bar(c_ref, lam, tl, ul, rel_c)
    assert (err <= bar).all(), (err / bar).max()
    rt, at = grad_tol(storage)
    excess = np.abs(grads - g_ref) - (rt * np.abs(g_ref) + at)
    assert excess.max() <= 0, excess.max()


def run_operator(acts_np, labels, tl, ul, storage, lam, weights=None, **kw):
    """rnnt_loss(reduction='none') forward + backward with per-utterance grad_output `weights`."""
    from warprnnt_pytorch import rnnt_loss
    x = torch.tensor(acts_np, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = rnnt_loss(x, lab, tl_, ul_, reduction='none', delay_penalty=f32(lam), **kw)
    w = torch.ones_like(out) if weights is None else torch.as_tensor(weights).to(out)
    (out * w).sum().backward()
    torch.cuda.synchronize()
    used = x.detach().double().cpu().numpy()      # the logits as stored (16-bit: rounded)
    return out.detach().double().cpu().numpy(), x.grad.double().cpu().numpy(), used


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_against_reference(shape, storage):
    N, T, U, V = SHAPES[shape]
    acts, labels, tl, ul = make(1, N, T, U, V)
    lam = 0.3
    w = np.linspace(0.5, 1.5, N)
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, lam, w)
    c_ref, g_ref = dr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam))
    assert_close(costs, grads, c_ref, g_ref * w[:, None, None, None], lam, tl, ul, storage)


@pytest.mark.parametrize("storage", ["fp32", "fp64"])
def test_positive_factors_and_negative_costs(storage):
    """lambda (T_b - 1)/2 well above |log p|: positive label log-factors, positive log-likelihoods, negative costs."""
    N, T, U, V = 3, 40, 6, 28
    acts, labels, tl, ul = make(2, N, T, U, V)
    lam = 2.0
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, lam)
    c_ref, g_ref = dr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam))
    assert (c_ref < 0).any()
    assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage)


@pytest.mark.parametrize("storage", STORAGES)
def test_fastemit_and_clamp_on_top(storage):
    N, T, U, V = SHAPES["tile"]
    acts, labels, tl, ul = make(3, N, T, U, V)
    lam, fe, clamp = 0.4, 0.3, 0.015625   # clamp exact in float32: fp64 calls see it rounded
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, lam, fastemit_lambda=f32(fe), clamp=clamp)
    c_ref, g_ref = dr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam), fastemit_lambda=f32(fe), clamp=clamp)
    assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage)
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, lam, fastemit_lambda=f32(fe))
    c_ref, g_ref = dr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam), fastemit_lambda=f32(fe))
    assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage)


@pytest.mark.parametrize("storage", ["fp32", "fp64"])
def test_tunv_layout_and_full_call(storage):
    """The full call, [N,T,U,V] and [T,U,N,V], against the forward / backward split, and the reference."""
    from warprnnt_pytorch import warp_rnnt
    N, T, U, V = SHAPES["chunk"]
    acts, labels, tl, ul = make(4, N, T, U, V)
    lam = 0.25
    costs, grads, used = run_operator(acts, labels, tl, ul, storage, lam)
    x = torch.tensor(acts, device="cuda", dtype=TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    c_full = torch.empty(N, device="cuda", dtype=x.dtype)
    g_full = torch.empty_like(x)
    ws = warp_rnnt.gpu_rnnt_async(x, lab, tl_, ul_, c_full, g_full, 0, delay_penalty=f32(lam))
    xt = x.permute(1, 2, 0, 3).contiguous()
    c_t = torch.empty(N, device="cuda", dtype=x.dtype)
    g_t = torch.empty_like(xt)
    ws2 = warp_rnnt.gpu_rnnt_async_tunv(xt, lab, tl_, ul_, c_t, g_t, 0, delay_penalty=f32(lam))
    torch.cuda.synchronize()
    del ws, ws2
    assert np.array_equal(c_full.double().cpu().numpy(), costs)
    assert np.array_equal(g_full.double().cpu().numpy(), grads)
    assert np.array_equal(c_t.double().cpu().numpy(), costs)
    assert np.array_equal(g_t.permute(2, 0, 1, 3).double().cpu().numpy(), grads)
    c_ref, g_ref = dr.dense_loss(used, labels, tl, ul, delay_penalty=f32(lam))
    assert_close(costs, grads, c_ref, g_ref, lam, tl, ul, storage)


@pytest.mark.parametrize("storage", STORAGES)
def test_nan_prefilled_gradients_zero_on_padding(storage):
    from warprnnt_pytorch import warp_rnnt
    N, T, U, V = SHAPES["tile"]
    acts, labels, tl, ul = make(5, N, T, U, V)
    tl[1], ul[1] = 3, 1
    x = torch.tensor(acts, device="cuda").to(TORCH[storage])
    lab, tl_, ul_ = cuda(labels, tl, ul)
    costs = torch.empty(N, device="cuda", dtype=warp_rnnt.costs_dtype(x))
    ws = warp_rnnt.gpu_rnnt_forward(x, lab, tl_, ul_, costs, 0, delay_penalty=0.5)
    grads = torch.full_like(x, float("nan"))
    warp_rnnt.gpu_rnnt_backward(x, lab, tl_, ul_, grads, None, 0, 1.0, ws, delay_penalty=0.5)
    g = grads.double().cpu().numpy()
    for b in range(N):
        assert np.isfinite(g[b, :tl[b], :ul[b] + 1]).all()
        assert (g[b, tl[b]:] == 0).all() and (g[b, :, ul[b] + 1:] == 0).all()


def test_zero_penalty_is_the_plain_entry_bitwise():
    from warprnnt_pytorch import rnnt_loss
    N, T, U, V = SHAPES["tile"]
    acts, labels, tl, ul = make(6, N, T, U, V)
    for storage in STORAGES:
        a = run_operator(acts, labels, tl, ul, storage, 0.0)
        x = torch.tensor(acts, device="cuda").to(TORCH[storage]).requires_grad_(True)
        lab, tl_, ul_ = cuda(labels, tl, ul)
        out = rnnt_loss(x, lab, tl_, ul_, reduction='none')
        out.sum().backward()
        assert np.array_equal(a[0], out.detach().double().cpu().numpy())
        assert np.array_equal(a[1], x.grad.double().cpu().numpy())
    # the *_lat C entries themselves at lambda = 0 against the entries without lattice options
    from warprnnt_pytorch import warp_rnnt
    lib = warp_rnnt.lib()
    x = torch.tensor(acts, device="cuda")
    lab, tl_, ul_ = cuda(labels, tl, ul)
    opt = warp_rnnt._options(x, 0)
    outs = []
    for use_lat in (False, True):
        c = torch.empty(N, device="cuda")
        g = torch.empty_like(x)
        ws = torch.empty(warp_rnnt.workspace_size(T, U, N), dtype=torch.uint8, device="cuda")
        args = (0, 0, x.data_ptr(), g.data_ptr(), lab.data_ptr(), ul_.data_ptr(), tl_.data_ptr(), V, N, c.data_ptr(),
                1.0, warp_rnnt.rnntGradOptions())
        st = (lib.rnnt_b200_loss_async_lat(*args, warp_rnnt.rnntLatticeOptions(0.0), ws.data_ptr(), opt) if use_lat
              else lib.rnnt_b200_loss_async_ex(*args, ws.data_ptr(), opt))
        assert st == 0
        torch.cuda.synchronize()
        outs.append((c.cpu(), g.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


# ---- pruned ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", STORAGES)
def test_pruned_full_windows_are_the_dense_loss_bitwise(storage):
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, V = SHAPES["chunk"]
    acts, labels, tl, ul = make(7, N, T, U, V)
    lam = 0.3
    costs, grads, _ = run_operator(acts, labels, tl, ul, storage, lam)
    x = torch.tensor(acts, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    ranges = torch.zeros(N, T, dtype=torch.int32, device="cuda")
    out = pruned_rnnt_loss(x, lab, tl_, ul_, ranges, reduction='none', delay_penalty=f32(lam))
    out.sum().backward()
    assert np.array_equal(out.detach().double().cpu().numpy(), costs)
    assert np.array_equal(x.grad.double().cpu().numpy(), grads)


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("V", [28, 500])
def test_pruned_against_reference(storage, V):
    from warprnnt_pytorch import pruned_rnnt_loss
    N, T, U, R = 4, 12, 7, 3
    rng = np.random.default_rng(8)
    _, labels, tl, ul = make(8, N, T, U, 2)
    labels = rng.integers(1, V, size=labels.shape).astype(np.int32)
    ranges = pr.random_monotone_ranges(rng, tl, ul, T, R)
    logits = (rng.standard_normal((N, T, R, V)) * 1.5).astype(np.float32)
    lam = 0.4
    x = torch.tensor(logits, device="cuda").to(TORCH[storage]).requires_grad_(True)
    lab, tl_, ul_, rg = cuda(labels, tl, ul, ranges)
    out = pruned_rnnt_loss(x, lab, tl_, ul_, rg, reduction='none', delay_penalty=f32(lam), fastemit_lambda=0.25)
    w = torch.linspace(0.5, 1.5, N, device="cuda").to(out)
    (out * w).sum().backward()
    c_ref, g_ref = dr.loss(x.detach().double().cpu().numpy(), labels, tl, ul, ranges, delay_penalty=f32(lam),
                           fastemit_lambda=0.25)
    assert_close(out.detach().double().cpu().numpy(), x.grad.double().cpu().numpy(), c_ref,
                 g_ref * w.double().cpu().numpy()[:, None, None, None], lam, tl, ul, storage)


# ---- additive joint ----------------------------------------------------------------------------------------------
def joint_inputs(seed, N, T, U, V):
    rng = np.random.default_rng(seed)
    trans = (rng.standard_normal((N, T, V)) * 1.5).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * 1.5).astype(np.float32)
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    return trans, pred, labels, tl, ul


def run_joint(trans, pred, labels, tl, ul, lam, lm=0.0, am=0.0, weights=None, **kw):
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    out = add_joint_rnnt_loss(tt, pp, lab, tl_, ul_, 0, 'none', lm_only_scale=lm, am_only_scale=am,
                              delay_penalty=f32(lam), **kw)
    w = torch.ones_like(out) if weights is None else torch.as_tensor(weights, dtype=torch.float32).cuda()
    (out * w).sum().backward()
    torch.cuda.synchronize()
    return out.detach().double().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy()


def assert_joint(costs, dF, dG, c_ref, dF_ref, dG_ref, labels, tl, ul, lam, scale, floor_dense=1e-9):
    err = np.abs(costs - c_ref)
    bar = cost_bar(c_ref, lam, tl, ul, 1e-5)
    assert (err <= bar).all(), (err / bar).max()
    s = np.asarray(scale, np.float64)[:, None, None]
    problems = grad_mismatch(dF, dF_ref * s, tl, labels, ul, 0, "dF", floor_dense=floor_dense) + \
        grad_mismatch(dG, dG_ref * s, ul + 1, labels, ul, 0, "dG", floor_dense=floor_dense)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("shape", [(3, 20, 7, 64), (2, 30, 40, 131), (3, 40, 9, 1024)],
                         ids=lambda s: "N%d_T%d_U%d_V%d" % s)
def test_joint_matches_the_dense_loss_on_materialised_logits(shape):
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N, T, U, V = shape
    trans, pred, labels, tl, ul = joint_inputs(9, N, T, U, V)
    lam = 0.3
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tl_, ul_ = cuda(labels, tl, ul)
    j = AddJointRNNTLoss(reduction='none', delay_penalty=f32(lam))(tt, pp, lab, tl_, ul_)
    j.sum().backward()
    acts = (tt.detach().double().unsqueeze(2) + pp.detach().double().unsqueeze(1)).requires_grad_(True)
    d = RNNTLoss(reduction='none', delay_penalty=f32(lam))(acts, lab, tl_, ul_)   # fp64 dense path
    d.sum().backward()
    assert_joint(j.detach().double().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy(),
                 d.detach().cpu().numpy(), acts.grad.sum(2).cpu().numpy(), acts.grad.sum(1).cpu().numpy(),
                 labels, tl, ul, lam, np.ones(N))


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("fe", [0.0, 0.3])
def test_joint_against_reference(lm, am, fe):
    N, T, U, V = 3, 24, 8, 131
    trans, pred, labels, tl, ul = joint_inputs(10, N, T, U, V)
    lam = 0.3
    w = np.linspace(0.5, 1.5, N)
    got = run_joint(trans, pred, labels, tl, ul, lam, lm, am, w, fastemit_lambda=f32(fe))
    want = dr.joint_reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul, lm, am,
                              delay_penalty=f32(lam), fastemit_lambda=f32(fe), scale=w)
    assert_joint(*got, *want, labels, tl, ul, lam, np.ones(N), floor_dense=1e-7 if am > 0 else 1e-9)


@pytest.mark.parametrize("lm,am", [(0.0, 0.0), (0.25, 0.0)])
def test_joint_ranges_from_the_penalised_lattice(lm, am):
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    N, T, U, V, R, lam = 4, 30, 9, 64, 3, 0.2
    for seed in range(20, 80):
        trans, pred, labels, tl, ul = joint_inputs(seed, N, T, U, V)
        occ = dr.joint_occupancies(trans, pred, labels, tl, ul, lm, am, delay_penalty=f32(lam))
        want, margin = pr.prune_ranges(occ, T, R)
        plain, _ = pr.prune_ranges(dr.joint_occupancies(trans, pred, labels, tl, ul, lm, am), T, R)
        if margin > 1e-4 and not np.array_equal(want, plain):
            break
    assert margin > 1e-4, "no seed with unambiguous windows"
    tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
    loss, ranges = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, R, reduction='none', lm_only_scale=lm,
                                                   am_only_scale=am, delay_penalty=f32(lam))
    got = ranges.cpu().numpy()
    assert np.array_equal(got, want)
    pr.check_range_properties(got, tl, ul, R)
    c_ref = dr.joint_costs(trans, pred, labels, tl, ul, lm, am, delay_penalty=f32(lam))
    assert (np.abs(loss.detach().double().cpu().numpy() - c_ref) <= cost_bar(c_ref, lam, tl, ul, 1e-5)).all()


def test_joint_zero_penalty_is_the_plain_entry_bitwise():
    from warprnnt_pytorch import add_joint_rnnt_loss_with_ranges
    from warprnnt_pytorch import warp_rnnt
    from warprnnt_pytorch.joint import joint_forward_call, rnntSmoothOptions
    N, T, U, V = 3, 20, 7, 64
    trans, pred, labels, tl, ul = joint_inputs(11, N, T, U, V)
    for lm, am in ((0.0, 0.0), (0.25, 0.1)):
        tt, pp, lab, tl_, ul_ = cuda(trans, pred, labels, tl, ul)
        smooth = rnntSmoothOptions(lm, am) if lm or am else None
        c0, c1 = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
        joint_forward_call(tt, pp, lab, tl_, ul_, c0, True, 0, smooth)
        joint_forward_call(tt, pp, lab, tl_, ul_, c1, True, 0, smooth, warp_rnnt.rnntLatticeOptions(0.0))
        assert torch.equal(c0, c1)
        _, r0 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, lm_only_scale=lm, am_only_scale=am)
        _, r1 = add_joint_rnnt_loss_with_ranges(tt, pp, lab, tl_, ul_, 2, lm_only_scale=lm, am_only_scale=am,
                                                delay_penalty=0.0)
        assert torch.equal(r0, r1)


# ---- batch groups and tuning hooks (child processes: the hooks are read once per process) -------------------------
def child(args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, os.path.join(HERE, "delay_hook_child.py")] + args, env=e,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_grouped_schedule_is_bitwise_the_ungrouped_call():
    out = child(["groups"], {"RNNT_B200_GROUPS": "4"})
    assert "groups ok" in out, out


def _hook_cases():
    from test_gpu_tuning_hooks import CASES
    return ["default"] + sorted({tuple(sorted(env.items())) for _, env, _, _, _ in CASES.values()})


PLAIN = re.compile(r"(rowstats_(chunk|tile|row)|grad_(chunk|tile|row)|joint_stats)_kernel<")
TWINS = ("rowstats_chunk_delay_kernel<float, 2, 256, true>", "grad_chunk_delay_kernel<float, 2, 256, false, false, true>",
         "rowstats_chunk_delay_kernel<float, 2, 256, false>", "grad_chunk_delay_kernel<float, 2, 256, false, false, false>",
         "joint_stats_delay_kernel<false>")


@pytest.mark.parametrize("hook", _hook_cases(), ids=lambda h: h if isinstance(h, str) else
                         "_".join("%s=%s" % (k[len("RNNT_B200_"):], v) for k, v in h))
def test_tuning_hooks(hook):
    """Every hook setting of test_gpu_tuning_hooks.CASES, one process each: the dense, pruned and joint shapes of
    hook_cases.py with a penalty match the reference, and only the penalised instantiations of the streaming and
    joint-statistics kernels ran."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("RNNT_B200_")}
    if hook != "default":
        env.update(dict(hook))
    r = subprocess.run([sys.executable, os.path.join(HERE, "delay_hook_child.py"), "hooks"], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    rep = json.loads(r.stdout.strip().splitlines()[-1])
    assert not rep["problems"], rep["problems"]
    kernels = [norm(k) for k in rep["kernels"]]
    assert not [k for k in kernels if PLAIN.search(k)], [k for k in kernels if PLAIN.search(k)]
    assert any("_delay_kernel<" in k for k in kernels)
    if hook == "default":
        for twin in TWINS:
            assert any(twin in k for k in kernels), (twin, [k for k in kernels if "delay" in k])
